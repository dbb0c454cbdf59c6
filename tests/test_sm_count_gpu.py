"""GPU: the stage-1 engine planned for sm_90 parts with fewer SMs than the H100 SXM's 132 (H100 PCIe 114, H20 78, MIG
slices fewer).  mvb_test_set_sm_limit(G) makes every engine created under it plan for G SMs: the persistent kernel runs
G CTAs with the K splits, attention units and fused-sampler choice of a G-SM part, and every split-K GEMM plans for G.
The limit only lowers the count, so every CTA stays co-resident and the run stands for that part.  Each G is capped at
this device's own count.  The limit is set only inside `sm_limit` and always cleared.

  path choice  1-layer production-width and tiny engines, every G, n_utts 1 .. 8, fp32 / bf16 KV, block_size 256 /
               2048: the body mvb_s1_decode runs (from the launch count) equals the mirror of test_sm_count_cpu.py
               (pc_ok, pc_att_fits, the owner guard 2 n_utts - 1 <= G, the fused-sampler condition).
  path A       k_gemv (bf16, and the LayerNorm architecture), k_gemv_w8, k_gemv_w4, k_gemv_f8: decode logits
               bit-identical to the uncapped engine.  A warp's products and their order depend only on its item, not on
               how many warps the grid has (gemv_grid only changes how many items a warp takes); a k_gemv_f8 block's sum
               does not depend on which CTA owns it (f8_gemv_ctas only changes how many blocks a CTA takes);
  fp8          test_fp8_gemv_gpu.py's float64 GEMV cases at G = 114, 78, 60, 54, 16, where a CTA owns 2 or 3 of wo's and
               w2's 16-row blocks and (from G = 80 down) lm_head's ragged tail block is a CTA's third (a mirror of
               f8_gemv_ctas); fp8 decode takes the widened rows path only above 8 slots, at every G;
  path C / B   the projection probes of test_decode_linear_ops_gpu.py (every phase at l* = 0, 12, 23, fp32 and bf16
               forms of the persistent kernel at every G for the batches path C takes there; path B's tensor-core rows
               path at G = 114, 60, 16) with that module's float64 references and bounds, the K splits from the
               plan_pc / plan_gemm mirrors at G;
               the attention of test_attention_ops_gpu.py at L = 2048 for the largest batch the tile table takes at G,
               its split merge above four splits and the fused 28 -> 40 burst;
  sampler      test_sampler_ops_gpu.py's supplied-noise burst and flat-tie order at G = 131, 114, 81 (fused: 20, 23
               and 32 vocabulary entries per CTA) and 80 (the host declines the fused sampler);
  G + 1 rows   the tiny model's path C at G = 3 / 7 with 2 / 4 utterances (one row more than CTAs) vs the float64 oracle;
  front end    at G = 114, 60, 16: test_stage1_frontend_ops_gpu.py's bit-exact embedding (paths B, C), staged layer-0
               operand and the S = 65 / 129 chunked prefill (plan_gemm's automatic split at G);
  stage 2      mvb_s2_forward at B = 3 (tiny and full) at G = 114, 60, 16 vs the float64 oracle port, graph = eager;
  end to end   at G = 114: the 1.2 B golden with a bf16 cache within the reference's own gap; EnCodec decode bit-identical
               to the uncapped engine (n_sm only feeds its co-residency check)."""
import contextlib
import ctypes as C

import pytest
import torch

import test_attention_ops_gpu as att
import test_decode_linear_ops_gpu as dl
import test_sampler_ops_gpu as smp
import test_stage1_frontend_ops_gpu as fe
import test_stage1_gpu as s1
import test_stage2_gpu as s2
from mvb200 import synth
from test_sm_count_cpu import FULL, SM_COUNTS, TINY, TINY_SM_COUNTS, att_tiles, body as body_mirror

pytestmark = pytest.mark.gpu

# launches of one mvb_s1_decode step on a 1-layer engine (k_identity_slots included): the fused persistent kernel once;
# persistent + k_sample; path A (embed + 5 + head) + k_sample; path B (rows + embed + 9 + head 2) + k_sample
DECODE_LAUNCHES = {"C-fused": 2, "C": 3, "A": 1 + 7 + 1, "B": 1 + 13 + 1}
PB_SM = [114, 60, 16]                     # the tensor-core rows path, the front end, prefill and stage 2


def _real():
    return torch.cuda.get_device_properties(0).multi_processor_count


def counts(gs):
    """The distinct counts min(G, this device's) of gs, in order."""
    out = []
    for g in gs:
        g = min(g, _real())
        if g not in out:
            out.append(g)
    return out


@contextlib.contextmanager
def sm_limit(n):
    from mvb200 import _lib
    lib = _lib.load()
    _lib.check(lib.mvb_test_set_sm_limit(n))
    try:
        yield min(n, _real())
    finally:
        _lib.check(lib.mvb_test_set_sm_limit(0))


def _state_dict(dims, std=0.0, seed=0):
    """1-layer stage-1 state dict of dims (D, H, F, V): all zero, or N(0, std^2) weights, N(0, 1) embeddings and gains
    near 1."""
    D, _, F, V = dims
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s, sd=std: torch.randn(*s, generator=g) * sd if std else torch.zeros(*s)  # noqa: E731
    gain = lambda: 1 + rnd(D, sd=0.1) if std else torch.ones(D)  # noqa: E731
    sd = {"transformer.wtes.0.weight": rnd(V, D, sd=1.0), "transformer.wpe.weight": rnd(2048, D, sd=1.0),
          "speaker_cond_pos.weight": rnd(D, 256), "transformer.ln_f.weight": gain(), "lm_heads.0.weight": rnd(V, D),
          "transformer.h.0.ln_1.weight": gain(), "transformer.h.0.attn.c_attn.weight": rnd(3 * D, D),
          "transformer.h.0.attn.c_proj.weight": rnd(D, D), "transformer.h.0.ln_2.weight": gain(),
          "transformer.h.0.mlp.swiglu.w1.weight": rnd(F, D), "transformer.h.0.mlp.swiglu.w3.weight": rnd(F, D),
          "transformer.h.0.mlp.c_proj.weight": rnd(D, F)}
    return {k: v.to(torch.bfloat16) for k, v in sd.items()}


def _engine(sd, dims, block, kv, utts, tc=None, mode=None, norm="rmsnorm"):
    from mvb200.fast_model import ModelArgs, Transformer
    D, H, F, V = dims
    n_layer = len({k.split(".")[2] for k in sd if k.startswith("transformer.h.")})
    cfg = ModelArgs(block_size=block, vocab_size=V, n_layer=n_layer, n_head=H, dim=D, intermediate_size=F, norm_type=norm)
    sd = {k: (v[:block] if k == "transformer.wpe.weight" else v) for k, v in sd.items()}
    m = Transformer.from_state_dict(sd, cfg, device="cuda:0", quantisation_mode=mode)
    m.setup_caches(2 * utts, block, kv_dtype=kv, tensor_core_path=tc)
    return m


def _begin(m, n, pos, tok=1):
    from mvb200 import _lib
    sp = _lib.Sampling(1.0, 1.0, 0.0, 0, 9999, 1)
    for u in range(n):
        _lib.check(m._lib.mvb_s1_begin(m.handle, u, tok + 7 * u, pos[u] if isinstance(pos, list) else pos, C.byref(sp),
                                       None, None, m._stream()))


def _launches(m):
    return int(m._lib.mvb_s1_launch_count(m.handle))


# ---------------------------------------------------------------------------------------------------------------------
def _sweep(dims, gs, blocks):
    from mvb200 import _lib
    sd = _state_dict(dims)
    seen = {}
    for G in counts(gs):
        for block in blocks:
            for kv in ("fp32", "bf16"):
                with sm_limit(G):
                    m = _engine(sd, dims, block, kv, 8)
                    try:
                        for n in range(1, 9):
                            want = body_mirror(dims, G, n, kv, block)
                            _begin(m, n, 3)
                            n0 = _launches(m)
                            _lib.check(m._lib.mvb_s1_decode(m.handle, n, 1, m._stream()))
                            torch.cuda.synchronize()
                            got = _launches(m) - n0
                            assert got == DECODE_LAUNCHES[want], \
                                f"G={G} {kv} block={block} n={n}: {got} launches, the mirror says {want}"
                            seen.setdefault(want, set()).add((G, n))
                    finally:
                        m.close()
    return seen


def test_path_choice_production_width():
    seen = _sweep(FULL, SM_COUNTS, (256, 2048))
    print("path choice, production width: " + ", ".join(f"{b}: {len(v)} (G, n)" for b, v in sorted(seen.items())))
    if _real() >= 15:     # the owner guard's example: 8 utterances, bf16 cache, block_size 256 at G = 8 -> path B
        assert (8, 8) in seen["B"] and (8, 4) in seen["C"]


def test_path_choice_tiny_model():
    seen = _sweep(TINY, TINY_SM_COUNTS + SM_COUNTS, (256, 2048))
    print("path choice, tiny model: " + ", ".join(f"{b}: {len(v)} (G, n)" for b, v in sorted(seen.items())))
    assert (2, 2) in seen["B"] and (1, 1) in seen["C"]


# ---------------------------------------------------------------------------------------------------------------------
PATH_A = {"bf16": dict(), "layernorm": dict(norm="layernorm"), "int8": dict(mode="int8"), "int4": dict(mode="int4"),
          "fp8": dict(mode="fp8")}


@pytest.mark.parametrize("fmt", list(PATH_A))
def test_path_a_bit_identical(fmt):
    """Path A decode logits (1 and 3 utterances at mixed positions, random weights and a random KV cache) on every
    capped engine equal the uncapped engine's bit for bit."""
    from mvb200 import _lib
    sd = _state_dict(FULL, std=0.02, seed=3)
    kw = PATH_A[fmt]

    def logits(G):
        ctx = sm_limit(G) if G else contextlib.nullcontext()
        with ctx:
            m = _engine(sd, FULL, 256, "fp32", 3, tc="", **kw)
            try:
                g = torch.Generator(device="cuda").manual_seed(5)
                m._kv.view(torch.float32).copy_(torch.randn(m._kv.numel() // 4, generator=g, device="cuda"))
                out = []
                for n, pos in ((1, [200]), (3, [5, 100, 255])):
                    _begin(m, n, pos)
                    lg = torch.empty(2 * n, FULL[3], device="cuda")
                    n0 = _launches(m)
                    _lib.check(m._lib.mvb_s1_step_logits(m.handle, n, lg.data_ptr(), m._stream()))
                    torch.cuda.synchronize()
                    assert _launches(m) - n0 == 1 + 7, f"{fmt} G={G} n={n}: path A did not run"
                    out.append(lg)
                return out
            finally:
                m.close()

    ref = logits(0)
    assert all(torch.isfinite(r).all() for r in ref)
    for G in counts(SM_COUNTS):
        for r, got in zip(ref, logits(G)):
            assert torch.equal(r.view(torch.int32), got.view(torch.int32)), f"{fmt}: G={G} differs from the uncapped engine"
    print(f"path A {fmt}: logits at G = {counts(SM_COUNTS)} bit-identical to the uncapped engine")


def test_fp8_rows_path_only_above_8_slots():
    """A 1-layer production-width fp8 engine with the rows path enabled decodes 1 .. 8 slots on path A (one k_gemv_f8
    launch row) and 9 .. 12 on path B (which widens the layer first: one launch more than bf16's path B), at every G."""
    from mvb200 import _lib
    sd = _state_dict(FULL)
    want = {"A": DECODE_LAUNCHES["A"], "B": DECODE_LAUNCHES["B"] + 1}
    for G in counts(SM_COUNTS):
        with sm_limit(G):
            m = _engine(sd, FULL, 256, "fp32", 12, mode="fp8")
            try:
                for n in range(1, 13):
                    _begin(m, n, 3)
                    n0 = _launches(m)
                    _lib.check(m._lib.mvb_s1_decode(m.handle, n, 1, m._stream()))
                    torch.cuda.synchronize()
                    body = "B" if n > 8 else "A"
                    assert _launches(m) - n0 == want[body], f"fp8 G={G} n={n}: {_launches(m) - n0} launches, not path {body}'s"
            finally:
                m.close()
    print(f"fp8 decode at G = {counts(SM_COUNTS)}: path A at 1 .. 8 slots, path B at 9 .. 12")


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def arena():
    a = dl.Arena()
    yield a
    del a.buf
    torch.cuda.empty_cache()


def _projection_probes(arena, form, G):
    with sm_limit(G):
        e = dl.Engine(arena, form, n_sm=G)
        try:
            if e.body == "C":
                e.utts = tuple(n for n in e.utts if body_mirror(FULL, G, n, e.kv, dl.BLOCK) in ("C", "C-fused"))
            worst = nw = 0.0
            if not e.utts:
                return None
            for probe in dl.PROBES:
                for l in dl.LSTAR:
                    w, n, _ = dl.run_probe(arena, e, probe, l)
                    worst, nw = max(worst, w), max(nw, n)
            splits = ", ".join(f"{m} {dl.n_split(e.body, m, G)}" for m in dl.MATS)
            print(f"{form} G={G} n_utts={list(e.utts)} K splits {splits}: max |err|/bound {worst:.2e}, normwise {nw:.2e}; "
                  f"peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
            return worst
        finally:
            e.close()
            torch.cuda.empty_cache()


@pytest.mark.parametrize("form", ["C-fp32", "C-bf16"])
def test_persistent_projections(arena, form):
    for G in counts(SM_COUNTS):
        _projection_probes(arena, form, G)


def test_rows_path_projections(arena):
    for G in counts(PB_SM):
        _projection_probes(arena, "B", G)


# ---------------------------------------------------------------------------------------------------------------------
def _att_getter(G):
    cache = {}

    def get(H, form, utts, n_layer=1):
        key = (H, form, utts, n_layer)
        if key not in cache:
            for k in list(cache):
                cache.pop(k).close()
            torch.cuda.empty_cache()
            cache[key] = att.Probe(H, form, utts, seed=H, n_layer=n_layer, n_sm=G)
        return cache[key]
    return get, cache


def test_attention_at_capacity():
    """H = 16, L = 2048 for every utterance of the largest batch path C takes at G: at or just under 128 tiles per CTA."""
    for G in counts(SM_COUNTS):
        for form, kv in (("C-fp32", "fp32"), ("C-mma", "bf16")):
            ns = [n for n in range(1, 9) if att._pc_fits(n, 16, kv, G) and 2 * n - 1 <= G]
            if not ns:
                continue
            get, cache = _att_getter(G)
            with sm_limit(G):
                try:
                    p = get(16, form, ns[-1])
                    assert att.expected_body(p, ns[-1]) == "C"
                    # at or just under capacity: the next batch is over the table or has no owner for its last entry
                    tiles = att_tiles(G, ns[-1], 16, kv, 2048)[1]
                    assert tiles >= 64 and (ns[-1] == 8 or not att._pc_fits(ns[-1] + 1, 16, kv, G)
                                            or 2 * ns[-1] + 1 > G), (G, form, ns[-1], tiles)
                    w, nw = att.check_rows(p, att.run_decode(p, [2048] * ns[-1], "wide", seed=G), f"{form} G={G}")
                finally:
                    for v in cache.values():
                        v.close()
            print(f"{form} G={G}: {ns[-1]} x L=2048, {att_tiles(G, ns[-1], 16, kv, 2048)[1]} tiles per CTA: "
                  f"max |err|/bound {w:.2e}, normwise {nw:.2e}")


def test_split_merge_and_fused_burst():
    """test_split_merge_above_four_splits where G / 4 > 4 splits are possible, and the fused 28 -> 40 fp32 burst of
    1 and 8 utterances where path C takes them with the fused sampler (V = 512: G >= 16)."""
    for G in counts(SM_COUNTS):
        print(f"G={G}:")
        get, cache = _att_getter(G)
        with sm_limit(G):
            try:
                if G >= 20:
                    att.split_merge(get)
                for n in (1, 8):
                    p = get(2, "C-fp32", 8, n_layer=2)
                    if att.expected_body(p, n) == "C" and -(-p.V // G) <= 32:
                        att.fused_burst(get, "C-fp32", 28, 40, n)
            finally:
                for v in cache.values():
                    v.close()


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", [131, 114, 81, 80])
def test_fused_sampler_slots(G):
    G = min(G, _real())
    with sm_limit(G):
        p = smp.Probe(2562, 8, True, n_sm=G)
        try:
            for n in (1, 8):
                body = smp.burst_supplied_noise(p, n, None)
                assert body == ("fused" if -(-2562 // G) <= 32 else "C+k_sample"), (G, n, body)
        finally:
            p.close()
        p = smp.Probe(4096, 8, True, n_sm=G)
        try:
            print(f"flat tie order V=4096 on {G} SMs [{smp.flat_tie_order(p)}]: exact")
        finally:
            p.close()


# ---------------------------------------------------------------------------------------------------------------------
def test_tiny_path_c_with_more_rows_than_ctas():
    """Tiny model, fp32 cache, G = 3 with 2 utterances and G = 7 with 4: R = 2 n_utts = G + 1 rows on G CTAs (the owner
    guard holds: CTA 2 (n - 1) = G - 1 exists).  One step_logits of each utterance at position 0 (its own token and
    speaker) against the float64 oracle port, 1e-3 of max |ref| as in the tiny-model end-to-end tests."""
    from mvb200 import _lib
    from oracle import stage1_port as P
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    o = P.Stage1Oracle(sd, d.n_head, d.norm_eps, torch.float64, faithful_full_cache=False)
    for G, n in ((3, 2), (7, 4)):
        if G > _real():
            continue
        assert body_mirror(TINY, G, n, "fp32", 256) in ("C", "C-fused") and 2 * n == G + 1
        with sm_limit(G):
            m = _engine(sd, TINY, 256, "fp32", n)
            try:
                spks = [synth.synthetic_speaker(seed=40 + u) for u in range(n)]
                toks = [5 + 301 * u for u in range(n)]
                for u in range(n):
                    m.set_speaker(u, spks[u])
                sp = _lib.Sampling(1.0, 1.0, 0.0, 0, 9999, 1)
                for u in range(n):
                    _lib.check(m._lib.mvb_s1_begin(m.handle, u, toks[u], 0, C.byref(sp), None, None, m._stream()))
                lg = torch.empty(2 * n, d.vocab_size, device="cuda")
                n0 = _launches(m)
                _lib.check(m._lib.mvb_s1_step_logits(m.handle, n, lg.data_ptr(), m._stream()))
                torch.cuda.synchronize()
                assert _launches(m) - n0 == 1 + 1, f"G={G} n={n}: path C did not run"
            finally:
                m.close()
        worst = 0.0
        for u in range(n):
            o.setup_caches()
            ref = o.forward(torch.tensor([[toks[u]], [toks[u]]]), spks[u], torch.tensor([0]))[:, -1]
            err = float((lg[2 * u:2 * u + 2].double().cpu() - ref).abs().max() / ref.abs().max())
            worst = max(worst, err)
            assert err < 1e-3, f"G={G} n={n} utterance {u}: rel err {err:.2e}"
        print(f"tiny path C, {2 * n} rows on G={G} CTAs: rel err vs float64 oracle {worst:.2e}")


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fe_model():
    m = fe.Model()
    yield m
    m.arenas = None
    torch.cuda.empty_cache()


def _fe_getter(model, G):
    cur = {}

    def get(fmt, kv, tc, utts):
        key = (fmt, kv, tc, utts)
        if key not in cur:
            for k in list(cur):
                cur.pop(k).close()
            torch.cuda.empty_cache()
            cur[key] = fe.Eng(model, fmt, kv, tc, utts, n_sm=G)
        return cur[key]
    return get, cur


def test_front_end_and_prefill(fe_model):
    """test_stage1_frontend_ops_gpu.py at G = 114, 60, 16: the bit-exact embedding of paths B and C, the persistent
    kernel's staged layer-0 operand (fp32 / bf16 KV, those of 1 / 4 / 5 / 8 utterances path C takes at G, qkv K split
    from plan_pc at G) and the
    prefill at S = 65, 129 (64-token chunks on path B, plan_gemm's automatic split at G) against float64."""
    for G in counts(PB_SM):
        get, cur = _fe_getter(fe_model, G)
        with sm_limit(G):
            try:
                fe.embedding_bit_exact(fe_model, get, "B")
                for kv in ("fp32", "bf16"):
                    # the batches path C takes at G (8 fp32 utterances exceed the tile table below 128 SMs)
                    ns = [n for n in (1, 4, 5, 8) if body_mirror(FULL, G, n, kv, fe.BLOCK) in ("C", "C-fused")]
                    fe.embedding_bit_exact(fe_model, get, f"C-{kv}", ns)
                    fe.staged_operand(fe_model, get, kv, ns)
                fe.prefill_cases(get, "bf16", "bf16", [(65, 0), (129, 0)])
            finally:
                for v in cur.values():
                    v.close()
        print(f"  (front end and prefill above: G={G})")


@pytest.mark.parametrize("tag,dims", [("tiny", synth.S2_TINY), ("full", synth.S2_FULL)])
def test_stage2_forward(tag, dims):
    """mvb_s2_forward at B = 3 at G = 114, 60, 16 (every split-K GEMM planned for G) against the float64 oracle port of
    test_stage2_gpu.py within its 1e-4, and the captured graph equal to the eager launches bit for bit."""
    from mvb200.second_stage import SecondStage
    ck = s2._checkpoint(dims)
    o = s2._oracle(ck, dims)
    for G in counts(PB_SM):
        with sm_limit(G):
            graph = SecondStage(ck, device="cuda:0", max_batch=3)
            eager = SecondStage(ck, device="cuda:0", max_batch=3, cuda_graph=False)
            idx, spk = s2._utterances(graph, dims, 3)
            tg, lg = graph.forward_tokens(idx, spk, 1.0, 200, seed=3, return_logits=True)
            te, le = eager.forward_tokens(idx, spk, 1.0, 200, seed=3, return_logits=True)
        rel, nw = s2._rel_err(lg, o.forward(idx.long(), spk.double()), 3)
        print(f"stage-2 {tag} B=3 G={G}: logits rel err vs float64 oracle {float(rel.max()):.2e}")
        assert float(rel.max()) < s2.TOL
        assert torch.equal(lg, le) and torch.equal(tg, te), f"G={G}: graph and eager differ"
        del graph, eager, lg, le
        torch.cuda.empty_cache()


def test_full_golden_and_encodec_at_114():
    """The 1.2 B golden (stage1_full.npz) with a bf16 cache through the persistent kernel and the chunked prefill planned
    for 114 SMs, within the reference's own bf16-vs-fp32 gap; EnCodec decode on an engine created at 114 SMs
    bit-identical to the uncapped engine (there n_sm only feeds the co-residency check)."""
    from mvb200.fast_model import pack_arena
    from mvb200.vocoder import EncodecDecodeEngine
    G = min(114, _real())
    golden = fe.__file__.rsplit("/", 1)[0] + "/golden"
    arena, offsets = pack_arena(synth.stage1_state_dict(synth.FULL, 0), synth.FULL.n_layer)
    full_arena = (arena.cuda(), offsets)
    del arena
    with sm_limit(G):
        s1.full_bf16_kv_golden(golden, full_arena)
    del full_arena
    torch.cuda.empty_cache()
    _, sd = synth.encodec_model_and_state_dict(seed=0)
    codes = torch.randint(0, 1024, (8, 375), generator=torch.Generator().manual_seed(375))
    wav = EncodecDecodeEngine(sd, device="cuda:0", max_frames=512).decode(codes)
    with sm_limit(G):
        wav_g = EncodecDecodeEngine(sd, device="cuda:0", max_frames=512).decode(codes)
    assert torch.equal(wav.view(torch.int32), wav_g.view(torch.int32)), "EnCodec decode at 114 SMs differs"
    print(f"1.2B golden (bf16 KV) at G={G} within the reference's gap; EnCodec decode at G={G} bit-identical")
