"""GPU: the stage-1 front end and the prefill plumbing at production width (metavoice-1B: D = 2048, H = 16, F = 5632,
V = 2562, speaker dim SD = 256, block_size 2048): the speaker projection k_spk_proj (bf16, int8 and fp8), the embedding
sum of every decode body (k_embed on path A, k_embed_rows on path B, the owner CTA of the persistent kernel on path C), the
layer-0 operand every persistent CTA stages straight from the tables, and mvb_s1_forward's chunk loop (k_rows_prefill,
k_gather_last, k_set_input, the [2, S, V] all-positions copy, the sampler rows).

PROBE MODEL.  2 layers whose matrices are all zero, so each layer adds exactly 0 to x (the residual stream only gains
+0, which turns -0 into +0: x is compared as floats).  Token and position tables are random bf16 N(0, 1) with about 0.1 %
of the entries replaced by +-(64 .. 256); W_spk is random bf16 N(0, 1), the ln_f gain 1 + 0.1 N(0, 1), lm_head bf16
N(0, 1 / D), speakers fp32 N(0, 1) with a different one in every slot.  The bf16, int8 (quantize.pack_arena_int8:
every Linear per output channel, so W_spk and lm_head get bf16 row scales that are not powers of two), int4
(quantize.pack_arena_int4: the zero layer matrices packed, W_spk stored as its bf16 W_deq, lm_head bf16 since 2562 % 8
!= 0) and fp8 (quantize.pack_arena_fp8: e4m3 codes and non-power-of-two bf16 row scales; the engine widens W_spk's and
lm_head's codes once at create into f8_spk and w8_head) engines are built from the same state dict.  The fp8 speaker
projection runs k_spk_proj over f8_spk with the arena's row scales: codes written after create are never read, which
is checked; the quantised workspace tail (layer scratch, w8_head, f8_spk) is mirrored against
mvb_s1_{int4,int8,fp8}_workspace_bytes and its widened copies compared with the arena's codes.  The workspace is read through a Python mirror of make_layout
(csrc/stage1_engine.cu), whose end is checked against mvb_s1_workspace_bytes here and the pinned totals of
tests/test_workspace_layout_cpu.py.

1 SPEAKER PROJECTION (mvb_s1_set_speaker).  Lane l of output row j runs one fma chain over k = l, l + 32, ... (SD / 32
  terms), then a 5-level butterfly adds the lanes: every product passes through at most ceil(SD / 32) + 5 roundings, so
      |y^ - y| <= gamma_(ceil(SD/32)+5) sum_k |W_jk| |spk_k|,    gamma_n = n u / (1 - n u), u = 2^-23.
  int8 / fp8: the chain runs over the exact codes q (W = s q), and the bf16 row scale multiplies the sum once: the same
  gamma times s sum |q| |spk| (to first order; 1.01 gamma is used), + u |y| for the product.  The reference is float64
  of the very weights the engine holds (bf16 W, s q, the int4 arena's W_deq).  The spk slice is NaN-filled first: only
  slot u's D floats may change, and none may stay NaN.  Slots 0, 3, max_utts - 1; a zero speaker (exactly 0 out); a
  speaker with one component of 1e6.

2 EMBEDDING, bit exact.  All four sites compute fl(fl(te + pe) + sp) with the speaker term only on the conditioned row,
  so the reference is float32 (te + pe) + sp with sp the engine's own spk_proj, and the check is equality.  After one
  mvb_s1_step_logits x is read from the workspace: L.x (path A, at 1 and 3 utterances), L.b_x (path B, batch row order,
  at 2, 8, 40 and 64 utterances: R = 128 = RB_MAX), L.c_x (path C, at 1, 4, 5 and 8 utterances: all four
  <fp32|bf16, 16|32> instances).  The launch count names the body that ran.  Tokens 0, V - 1, 2048 (end of audio) and
  random ones, the unconditioned row's token different from the conditioned row's (written into row_tok after
  mvb_s1_begin); positions 0, 1, 63, 64, 2046, 2047 and random ones.

3 STAGED OPERAND of the persistent kernel.  Path C never writes layer 0's QKV operand: each CTA stages x g from the
  tables.  With layer 0's W_qkv = [0; I; 0] and a random ln_1 gain g, the appended k is rs * hilo(fl(x_staged g)).  It is
  compared with the reference built from the x the owner CTA wrote (read from L.c_x) with the operand and bound of
  tests/test_decode_linear_ops_gpu.py for path C, plus the sum of squares: x is not on a grid here, so the fp32 sum of
  squares is off by <= gamma_depth ss, depth = 8 (a thread's chunk) + 5 (warp) + 8 (shared-memory adds) + S (the split
  adds) + 2 (/ D, + eps), which moves rs by <= 0.51 depth u: + 0.51 depth u A.  A bf16 cache adds 2^-8 (|y| + bound).

4 PREFILL (mvb_s1_forward).  logits[c, s] against the float64 head (bf16 W, or s q for int8) applied to the RMSNorm of
  the bit-exact x of section 2, with the operand each body stages (path B: hilo(fl(fl(x rs) g)) by k_prep_b; path A:
  fl(fl(x rs) g) in fp32) and the bound lin_bound of tests/test_decode_linear_ops_gpu.py (the m16n8k16 model of
  tests/test_gemm_ops_gpu.py per split, the k-split from plan_gemm_ksplit: R = 2 Sc only changes the column count), + the
  sum of squares of x (k_prep_b and the GEMV prologue: 8-term chains, 5-level butterfly, 8 warp sums, / D, + eps:
  depth 24) and, for int8, u |y| for the row scale.  Lengths S in {1, 2, 63, 64, 65, 128, 129, 2047} at pos0 = 0 and
  S = 70 at pos0 in {1000, 1977}, into slot 0 and slot max_utts - 1 of an 8-slot engine, for bf16, int8, int4 and fp8
  with fp32 and bf16 KV (fp8 at S = 1 and on the path A loop: k_gemv_f8's head, the gamma of tests/test_fp8_gemv_gpu.py
  and its own sum-of-squares depth D / 32 + 12); S = 1 takes the one-position path A loop, the rest the 64-token chunks (the launch count shows which),
  and a CUDA-core-only engine runs the path A loop at S = 2 and 65.  Every call runs with all_positions = 1 into a
  caller buffer between NaN guards (every element written, nothing outside) and with all_positions = 0 (the 2 x V copy
  equals the slot's sampler rows, which must satisfy the bound of the last position).  Afterwards slot_map[0] = utt,
  pos[utt] = pos0 + S - 1, row_tok = the two rows' last tokens, and the row map of the last chunk (b_rows) is the chunk's.
  Isolation: the KV cache holds random values beforehand; only [pos0, pos0 + S) of the slot's two cache rows change (to
  the zero k, v of the zero layers), and the other slots' logits rows, every spk entry and the other slots' decode state
  are unchanged.

5 SENSITIVITY.  Altered references that must be caught: bit-exact checks must differ on >= 99 % of the affected
  elements (the speaker on the unconditioned row too, slot u - 1's speaker, the speaker rounded to bf16 before the add,
  the position row pos - 1); bounded checks must put >= 50 % of the affected elements over the bound (the int8 speaker
  projection without its row scale: >= 99 %, int8 / fp8 with each row's scale from its neighbour; prefill: the position row pos0 + s0 + s - 1, the chunk offset s0 dropped
  from the token index, the unconditioned tokens taken from row 0, slot u - 1's speaker, the speaker on both rows, the
  last-position gather from row Sc - 2; staged operand: the speaker dropped, the other row's token, the position row
  pos + 1)."""
import ctypes as C
import math

import pytest
import torch

from test_decode_linear_ops_gpu import U, lin_bound, operand, plan_gemm_ksplit, plan_pc

pytestmark = pytest.mark.gpu

D, H, F, V, NL, SPK, BLOCK = 2048, 16, 5632, 2562, 2, 256, 2048
EOA = 2048
BF16_U = 2.0 ** -8
SS_DEPTH_AB = 24           # sum of squares of k_prep_b and of the GEMV prologue (module docstring, section 4)
MAXU = 8                   # slots of the engines of sections 1, 3 and 4
# kernel launches of one mvb_s1_step_logits (k_identity_slots included) for the 2-layer model (as in
# tests/test_decode_linear_ops_gpu.py): A embed + 5 per layer + head; B rows + embed + 9 per layer + head; C one kernel
LAUNCHES = {"A": 1 + 1 + 5 * NL + 1, "B": 1 + 1 + 1 + 9 * NL + 2, "C": 1 + 1}
# body -> (kv dtype, tensor_core_path, slots, utterance counts, x buffer)
BODIES = {"A": ("fp32", "", 3, (1, 3), "x"), "B": ("bf16", "B", 64, (2, 8, 40, 64), "b_x"),
          "C-fp32": ("fp32", "BC", MAXU, (1, 4, 5, 8), "c_x"), "C-bf16": ("bf16", "BC", MAXU, (1, 4, 5, 8), "c_x")}
POS_EDGE = [0, 1, 63, 64, 2046, 2047]
TOK_EDGE = [0, V - 1, EOA]
PREFILL = [(S, 0) for S in (1, 2, 63, 64, 65, 128, 129, 2047)] + [(70, 1000), (70, 1977)]
BIT_SENS, BOUND_SENS = 0.99, 0.5


def gam(n):
    return n * U / (1 - n * U)


def tau_ss(depth):
    return 0.51 * depth * U


# ---------------------------------------------------------------------------------------------------------------------
# workspace: a mirror of make_layout (csrc/stage1_engine.cu)
def ws_layout(U_, n_layer=NL, dim=D, inter=F, vocab=V, n_head=H, block=BLOCK, spk_dim=SPK, max_new=None):
    """name -> (byte offset, bytes) of every slice of the stage-1 workspace, and "total"."""
    max_new = max_new or block
    R, RB, NBM = 2 * U_, 128, 256
    sc = 0
    for M, K, sw in ((3 * dim, dim, False), (dim, dim, False), (inter, dim, True), (dim, inter, False), (vocab, dim, False)):
        sc = max(sc, -(-M // 128) * plan_gemm_ksplit(M, K, 132) * (2 if sw else 1) * NBM * 128)   # plan_gemm at GEMM_MAX_SM
    sizes = [("x", R * dim * 4), ("qkv", R * 3 * dim * 4), ("att", R * dim * 4), ("ffn", R * inter * 4),
             ("logits", R * vocab * 4), ("spk", U_ * dim * 4), ("part_o", R * n_head * 8 * 128 * 4),
             ("part_ml", R * n_head * 8 * 2 * 4), ("slot_map", U_ * 4), ("pos", U_ * 4), ("row_tok", R * 4),
             ("done", U_ * 4), ("n_gen", U_ * 4), ("gen_tokens", U_ * max_new * 4), ("sampled", U_ * max_new * 4),
             ("samp", U_ * 32), ("noise", U_ * 8), ("forced", U_ * 8), ("ticket", R * n_head * 4), ("budget", U_ * 4),
             ("noise_base", U_ * 4), ("stage_idx", U_ * 2 * block * 4), ("stage_spk", U_ * spk_dim * 4),
             ("stage_forced", U_ * max_new * 4), ("stage_noise", U_ * 32 * vocab * 4),
             ("b_x", RB * dim * 4), ("b_qkv", RB * 3 * dim * 4), ("b_att", RB * dim * 4), ("b_ffn", RB * inter * 4),
             ("b_logits", RB * vocab * 4), ("b_last", 2 * dim * 4), ("b_B", NBM * max(inter, dim) * 2),
             ("b_rows", 5 * RB * 4), ("b_scratch", sc * 4), ("b_tickets", 256 * 4),
             ("b_part_o", RB * n_head * 8 * 128 * 4), ("b_part_ml", RB * n_head * 8 * 2 * 4),
             ("b_att_tickets", RB * n_head * 4),
             ("c_x", 16 * dim * 4), ("c_qkv", 16 * 3 * dim * 4), ("c_gu", 16 * 2 * inter * 4),
             ("c_part_o", 16 * n_head * 64 * 128 * 4), ("c_part_ml", 16 * n_head * 64 * 2 * 4), ("c_bar", 256),
             ("c_trace", 160 * 512 * 8), ("c_stat", (2 * n_layer + 1) * 16 * 4), ("c_samp_part", 8 * 256 * 4),
             ("c_samp_best", 2 * 8 * 8)]
    off, out = 0, {}
    for name, n in sizes:
        out[name] = (off, n)
        off = (off + n + 255) // 256 * 256
    out["total"] = off
    return out


def test_workspace_mirror():
    """The mirror ends where the pinned mvb_s1_workspace_bytes totals do."""
    from mvb200 import synth
    from test_workspace_layout_cpu import S1_BYTES
    dims = {"full": synth.FULL, "tiny": synth.TINY}
    for (name, utts, _), (want, _) in S1_BYTES.items():
        d = dims[name]
        got = ws_layout(utts, d.n_layer, d.dim, d.intermediate_size, d.vocab_size, d.n_head, d.block_size,
                        d.speaker_emb_dim)["total"]
        assert got == want, (name, utts, got, want)


def quant_tail(lay, dim=D, inter=F, vocab=V, spk_dim=SPK):
    """Mirror of make_layout's quantised tail: the one-layer bf16 weight scratch (int4, int8, fp8), lm_head's widened q
    (int8, fp8: w8_head), speaker_cond_pos's widened q (fp8: f8_spk); name -> (byte offset, bytes), and the totals."""
    out, off = {}, lay["total"]
    for name, n in (("layer_scratch", (4 * dim * dim + 3 * dim * inter) * 2), ("w8_head", vocab * dim * 2),
                    ("f8_spk", dim * spk_dim * 2)):
        out[name] = (off, n)
        off = (off + n + 255) // 256 * 256
        out[{"layer_scratch": "int4", "w8_head": "int8", "f8_spk": "fp8"}[name]] = off
    return out


# ---------------------------------------------------------------------------------------------------------------------
class Model:
    """The probe state dict, its three device arenas, the tables and the per-slot speakers."""

    def __init__(self):
        from mvb200.fast_model import pack_arena
        from mvb200.quantize import pack_arena_fp8, pack_arena_int4, pack_arena_int8
        g = torch.Generator().manual_seed(0)

        def table(rows):
            t = torch.randn(rows, D, generator=g)
            big = torch.rand(rows, D, generator=g) < 1e-3
            mag = (64 + 192 * torch.rand(rows, D, generator=g)) * (torch.randint(0, 2, (rows, D), generator=g) * 2 - 1)
            return torch.where(big, mag, t).to(torch.bfloat16)

        bf = torch.bfloat16
        sd = {"transformer.wtes.0.weight": table(V), "transformer.wpe.weight": table(BLOCK),
              "speaker_cond_pos.weight": torch.randn(D, SPK, generator=g).to(bf),
              "transformer.ln_f.weight": (1 + 0.1 * torch.randn(D, generator=g)).to(bf),
              "lm_heads.0.weight": (torch.randn(V, D, generator=g) * D ** -0.5).to(bf)}
        for i in range(NL):
            p = f"transformer.h.{i}."
            sd.update({p + "ln_1.weight": torch.ones(D, dtype=bf), p + "ln_2.weight": torch.ones(D, dtype=bf),
                       p + "attn.c_attn.weight": torch.zeros(3 * D, D, dtype=bf),
                       p + "attn.c_proj.weight": torch.zeros(D, D, dtype=bf),
                       p + "mlp.swiglu.w1.weight": torch.zeros(F, D, dtype=bf),
                       p + "mlp.swiglu.w3.weight": torch.zeros(F, D, dtype=bf),
                       p + "mlp.c_proj.weight": torch.zeros(D, F, dtype=bf)})
        self.sd = sd
        self.arenas = {"bf16": pack_arena(sd, NL), "int8": pack_arena_int8(sd, NL)[:2], "int4": pack_arena_int4(sd, NL)[:2],
                       "fp8": pack_arena_fp8(sd, NL)[:2]}
        self.arenas = {k: (a.cuda(), o) for k, (a, o) in self.arenas.items()}
        self.tok = sd["transformer.wtes.0.weight"].cuda()
        self.pos = sd["transformer.wpe.weight"].cuda()
        self.gf = sd["transformer.ln_f.weight"].cuda()
        self.spks = torch.randn(64, SPK, generator=g).cuda()


class Eng:
    def __init__(self, model, fmt, kv, tc, utts, n_sm=None):
        """n_sm: the SM count the engine is planned for (default: this device's)."""
        from mvb200.fast_model import ModelArgs, Transformer
        from test_decode_linear_ops_gpu import _n_sm
        self.model, self.fmt, self.kv, self.tc, self.utts = model, fmt, kv, tc, utts
        self.n_sm = n_sm or _n_sm()
        arena, self.offsets = model.arenas[fmt]
        cfg = ModelArgs(block_size=BLOCK, vocab_size=V, n_layer=NL, n_head=H, dim=D, intermediate_size=F)
        self.m = Transformer(cfg, arena, self.offsets, device="cuda:0", quantisation_mode=None if fmt == "bf16" else fmt)
        self.m.setup_caches(2 * utts, BLOCK, kv_dtype=kv, tensor_core_path=tc)
        self.lib, self.h = self.m._lib, self.m.handle
        self.ws = self.m._ws[1]
        self.lay = ws_layout(utts)
        assert self.lib.mvb_s1_workspace_bytes(C.byref(self.m._cfg)) == self.lay["total"], "workspace mirror"
        self.dt = torch.float32 if kv == "fp32" else torch.bfloat16
        self.cache = self.m._kv.view(self.dt).view(NL, 2, 2 * utts, H, BLOCK, 128)
        self.arena = arena
        for name in ("transformer.wtes.0.weight", "transformer.wpe.weight", "transformer.ln_f.weight"):
            t = model.sd[name]
            assert torch.equal(self.tensor(name, t.shape, torch.bfloat16).cpu(), t), f"{fmt} arena: {name}"
        self.set_speakers()

    def tensor(self, name, shape, dtype, extra=0):
        from mvb200.fast_model import _GLOBAL_KEYS
        o = self.offsets[_GLOBAL_KEYS.index(name)] + extra
        n = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
        return self.arena[o:o + n].view(dtype).view(*shape)

    def weights(self, name, M, K):
        """float64 (W or q [M, K], row scale [M] or None) of a global Linear as the engine holds it."""
        if self.fmt in ("int8", "fp8"):
            if self.fmt == "int8":
                q = self.tensor(name, (M, K), torch.int8).double()
            else:
                from mvb200.quantize import unpack_fp8_codes
                q = unpack_fp8_codes(self.tensor(name, (M * K,), torch.uint8).cpu(), M, K).double().cuda()
            s = self.tensor(name, (M,), torch.bfloat16, extra=(M * K + 255) // 256 * 256).double()
            return q, s
        return self.tensor(name, (M, K), torch.bfloat16).double(), None

    def set_speakers(self):
        for u in range(self.utts):
            self.m.set_speaker(u, self.model.spks[u])
        torch.cuda.synchronize()

    def sl(self, name, dtype):
        o, n = self.lay[name]
        return self.ws[o:o + n].view(dtype)

    def launches(self):
        return int(self.lib.mvb_s1_launch_count(self.h))

    def st(self):
        return self.m._stream()

    def close(self):
        self.m.close()


@pytest.fixture(scope="module")
def model():
    m = Model()
    yield m
    m.arenas = None
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def engines(model):
    cur = {}

    def get(fmt, kv, tc, utts):
        key = (fmt, kv, tc, utts)
        if key not in cur:
            for k in list(cur):
                cur.pop(k).close()
            torch.cuda.empty_cache()
            cur[key] = Eng(model, fmt, kv, tc, utts)
        return cur[key]
    yield get
    for v in cur.values():
        v.close()


def over(got, ref, bound):
    return (got - ref).abs() > bound


def check_bound(label, got, ref, bound):
    err = (got - ref).abs()
    ratio = float((err / bound).max())
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, (f"{label}: {bad.shape[0]} elements over the bound (max ratio {ratio:.2e}); first "
                              f"{bad[0].tolist()}: got {float(got[tuple(bad[0])]):.9e}, want {float(ref[tuple(bad[0])]):.9e}")
    return ratio


def caught(label, frac, need):
    print(f"  sensitivity {label}: {100 * frac:.1f} % of the affected elements caught")
    assert frac >= need, f"a reference with {label} passes: only {100 * frac:.1f} % caught"


# ---------------------------------------------------------------------------------------------------------------------
# 1. speaker projection
@pytest.mark.parametrize("fmt", ["bf16", "int8", "int4", "fp8"])
def test_speaker_projection(model, engines, fmt):
    e = engines(fmt, "fp32", "BC", MAXU)
    W, s = e.weights("speaker_cond_pos.weight", D, SPK)
    if fmt in ("int8", "fp8"):
        from mvb200.quantize import quantize_fp8_per_channel, quantize_per_channel
        q0, s0 = (quantize_per_channel if fmt == "int8" else quantize_fp8_per_channel)(model.sd["speaker_cond_pos.weight"])
        assert torch.equal(W.cpu(), q0.double()) and torch.equal(s.cpu(), s0.double())
        assert not all(math.log2(v).is_integer() for v in s.abs().tolist()), f"{fmt} row scales are all powers of two"
    elif fmt == "int4":
        from mvb200.quantize import dequantize, group_quantize
        wd = dequantize(*group_quantize(model.sd["speaker_cond_pos.weight"]))
        assert torch.equal(W.cpu(), wd.double()) and not torch.equal(wd, model.sd["speaker_cond_pos.weight"])
    scale = torch.ones(D, dtype=torch.float64, device="cuda") if s is None else s
    g = torch.Generator(device="cuda").manual_seed(11)
    huge = torch.randn(SPK, generator=g, device="cuda")
    huge[77] = 1e6
    cases = [(0, torch.randn(SPK, generator=g, device="cuda")), (3, torch.randn(SPK, generator=g, device="cuda")),
             (MAXU - 1, torch.randn(SPK, generator=g, device="cuda")), (3, torch.zeros(SPK, device="cuda")), (MAXU - 1, huge)]
    spk = e.sl("spk", torch.float32).view(MAXU, D)
    worst = 0.0
    try:
        for u, vec in cases:
            spk.fill_(float("nan"))
            e.m.set_speaker(u, vec)
            torch.cuda.synchronize()
            got = spk.double()
            others = torch.arange(MAXU, device="cuda") != u
            assert torch.isnan(got[others]).all(), f"{fmt} slot {u}: spk entries of other slots written"
            assert not torch.isnan(got[u]).any(), f"{fmt} slot {u}: spk entries left unwritten"
            v64 = vec.double()
            y = (W @ v64) * scale
            A = (W.abs() @ v64.abs()) * scale
            b = 1.01 * gam(-(-SPK // 32) + 5) * A + (U * y.abs() if s is not None else 0) + 1e-300
            if not vec.any():
                assert (got[u] == 0).all(), f"{fmt}: a zero speaker projects to nonzero values"
            worst = max(worst, check_bound(f"{fmt} k_spk_proj slot {u}", got[u], y, b))
            if s is not None and u == 0:
                caught(f"{fmt} projection without its row scale", float(over(got[u], W @ v64, b).double().mean()), BIT_SENS)
                caught(f"{fmt} projection with each row's scale from its neighbour",
                       float(over(got[u], (W @ v64) * torch.roll(s, 1), b).double().mean()), BOUND_SENS)
    finally:
        e.set_speakers()
    print(f"k_spk_proj<{'int8_t' if fmt == 'int8' else 'bf16'}> ({fmt} engine): max |err|/bound {worst:.2e}")


def test_fp8_speaker_codes_widened_at_create(model, engines):
    """An fp8 engine projects the speaker through f8_spk, speaker_cond_pos's codes widened once at create: codes written
    into the arena afterwards are never read (the projection stays bit for bit what it was), while the row scales are
    read from the arena at every mvb_s1_set_speaker.  So W_spk is part of the engine: change it by creating a new one."""
    e = engines("fp8", "fp32", "BC", MAXU)
    o = e.offsets[2]
    codes = e.arena[o:o + D * SPK]
    scales = e.arena[o + (D * SPK + 255) // 256 * 256:][:2 * D].view(torch.bfloat16)
    spk = e.sl("spk", torch.float32).view(MAXU, D)
    vec = torch.randn(SPK, generator=torch.Generator(device="cuda").manual_seed(12), device="cuda")
    keep_c, keep_s = codes.clone(), scales.clone()
    try:
        e.m.set_speaker(1, vec)
        torch.cuda.synchronize()
        before = spk[1].clone()
        codes.copy_(torch.roll(keep_c, 1))                  # other codes, same scales
        e.m.set_speaker(1, vec)
        torch.cuda.synchronize()
        assert torch.equal(spk[1].view(torch.int32), before.view(torch.int32)), "fp8 k_spk_proj read the arena's codes"
        codes.copy_(keep_c)
        scales.mul_(2)                                      # the scales are live: exactly twice the projection
        e.m.set_speaker(1, vec)
        torch.cuda.synchronize()
        assert torch.equal(spk[1], 2 * before), "fp8 k_spk_proj did not apply the arena's row scales"
    finally:
        codes.copy_(keep_c)
        scales.copy_(keep_s)
        e.set_speakers()
    print("fp8 speaker projection: codes widened at create, row scales read at every set_speaker")


@pytest.mark.parametrize("fmt", ["int8", "fp8"])
def test_quant_workspace_mirror(model, engines, fmt):
    """mvb_s1_{int4,int8,fp8}_workspace_bytes end where the mirror's quantised tail does, and the widened copies the
    engine makes at create hold the arena's codes exactly: lm_head's in w8_head, and for fp8 speaker_cond_pos's in f8_spk."""
    e = engines(fmt, "fp32", "BC", MAXU)
    tail = quant_tail(e.lay)
    for f in ("int4", "int8", "fp8"):
        got = getattr(e.lib, f"mvb_s1_{f}_workspace_bytes")(C.byref(e.m._cfg))
        assert got == tail[f], (f, got, tail[f])
    assert e.ws.numel() >= tail[fmt]
    names = [("w8_head", "lm_heads.0.weight", V, D)] + ([("f8_spk", "speaker_cond_pos.weight", D, SPK)] if fmt == "fp8" else [])
    for slot, name, M, K in names:
        o, n = tail[slot]
        widened = e.ws[o:o + n].view(torch.bfloat16).view(M, K)
        q, _ = e.weights(name, M, K)
        assert torch.equal(widened.double(), q), f"{fmt} {slot}: the widened copy differs from the arena's {name} codes"
    print(f"{fmt} workspace: int4 / int8 / fp8 totals {tail['int4']} / {tail['int8']} / {tail['fp8']} bytes; "
          f"{', '.join(n[0] for n in names)} exact")


# ---------------------------------------------------------------------------------------------------------------------
# 2. embedding in every decode body
def design(n, seed):
    """Per utterance: (cond token, uncond token, position), covering the edge tokens and positions."""
    g = torch.Generator().manual_seed(seed)
    tc = [TOK_EDGE[i] if i < len(TOK_EDGE) else int(torch.randint(0, V, (1,), generator=g)) for i in range(n)]
    tu = [(t + 1 + int(torch.randint(0, V - 1, (1,), generator=g))) % V for t in tc]
    if n > 1:
        tu[1] = EOA if tc[1] != EOA else 0
    ps = [POS_EDGE[(i + seed) % len(POS_EDGE)] if i < len(POS_EDGE) else int(torch.randint(0, BLOCK, (1,), generator=g))
          for i in range(n)]
    return tc, tu, ps


def begin(e, n, tc, tu, ps):
    from mvb200 import _lib
    sp = _lib.Sampling(1.0, 1.0, 0.0, 0, 9999, 1)
    for u in range(n):
        _lib.check(e.lib.mvb_s1_begin(e.h, u, tc[u], ps[u], C.byref(sp), None, None, e.st()))
    rt = e.sl("row_tok", torch.int32)
    rt[1:2 * n:2] = torch.tensor(tu, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    assert e.sl("pos", torch.int32)[:n].tolist() == ps, "workspace mirror: pos"
    assert rt[0:2 * n:2].tolist() == tc, "workspace mirror: row_tok"


def step_x(e, n, body, xbuf):
    """One mvb_s1_step_logits for utterances [0, n); x [2 n, D] read from the body's buffer."""
    from mvb200 import _lib
    n0 = e.launches()
    lg = torch.full((2 * n + 2, V), float("nan"), device="cuda")
    _lib.check(e.lib.mvb_s1_step_logits(e.h, n, lg.data_ptr(), e.st()))
    torch.cuda.synchronize()
    assert e.launches() - n0 == LAUNCHES[body[0]], f"{body} n={n}: body {body[0]} did not run"
    assert torch.isnan(lg[2 * n:]).all() and not torch.isnan(lg[:2 * n]).any(), f"{body} n={n}: logits rows"
    return e.sl(xbuf, torch.float32).view(-1, D)[:2 * n].clone()


def x_rows(model, sp, toks, poss, slots, cond, *, spk_both=False, spk_shift=0, spk_bf16=False):
    """float32 x [R, D] = fl(fl(te + pe) + sp) (speaker on the conditioned rows), and the altered variants."""
    t = torch.as_tensor(toks, device="cuda").long()
    p = torch.as_tensor(poss, device="cuda").long()
    u = (torch.as_tensor(slots, device="cuda").long() - spk_shift) % sp.shape[0]
    c = torch.as_tensor(cond, device="cuda").bool()
    x = model.tok[t].float() + model.pos[p].float()
    s = sp[u]
    if spk_bf16:
        s = s.to(torch.bfloat16).float()
    on = torch.ones_like(c) if spk_both else c
    return torch.where(on[:, None], x + s, x)


def body_rows(n, tc, tu, ps):
    toks = [t for u in range(n) for t in (tc[u], tu[u])]
    poss = [ps[u] for u in range(n) for _ in range(2)]
    slots = [u for u in range(n) for _ in range(2)]
    cond = [c == 0 for _ in range(n) for c in range(2)]
    return toks, poss, slots, cond


@pytest.mark.parametrize("body", list(BODIES))
def test_embedding_bit_exact(model, engines, body):
    embedding_bit_exact(model, engines, body)


def embedding_bit_exact(model, engines, body, counts=None):
    """test_embedding_bit_exact on the engines `engines` returns (their SM count may be capped), for the utterance
    counts `counts` (default: the body's own) that the body takes on that count."""
    kv, tc_path, utts, own, xbuf = BODIES[body]
    counts = counts or own
    e = engines("bf16", kv, tc_path, utts)
    e.m._kv.zero_()
    sp = e.sl("spk", torch.float32).view(utts, D).clone()
    for n in counts:
        tc, tu, ps = design(n, n)
        begin(e, n, tc, tu, ps)
        got = step_x(e, n, body, xbuf)
        rows = body_rows(n, tc, tu, ps)
        ref = x_rows(model, sp, *rows)
        eq = got == ref
        assert eq.all(), f"{body} n={n}: {int((~eq).sum())} elements of x differ from fl(fl(te + pe) + sp)"
        cond = torch.tensor(rows[3], device="cuda")
        if n == counts[-1]:
            unc = ~cond
            caught(f"{body}: speaker on both rows", float((got != x_rows(model, sp, *rows, spk_both=True))[unc].float().mean()), BIT_SENS)
            caught(f"{body}: speaker rounded to bf16", float((got != x_rows(model, sp, *rows, spk_bf16=True))[cond].float().mean()), BIT_SENS)
            if n > 1:
                sel = cond & (torch.tensor(rows[2], device="cuda") > 0)
                caught(f"{body}: slot u - 1's speaker", float((got != x_rows(model, sp, *rows, spk_shift=1))[sel].float().mean()), BIT_SENS)
            pm = [max(p - 1, 0) for p in rows[1]]
            sel = torch.tensor(rows[1], device="cuda") > 0
            caught(f"{body}: position row pos - 1", float((got != x_rows(model, sp, rows[0], pm, rows[2], rows[3]))[sel].float().mean()), BIT_SENS)
    print(f"embedding, body {body} ({LAUNCHES[body[0]]} launches), n_utts {list(counts)}, {e.n_sm} SMs: bit exact")


# ---------------------------------------------------------------------------------------------------------------------
# 3. the persistent kernel's staged layer-0 operand
@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_staged_operand(model, engines, kv):
    staged_operand(model, engines, kv)


def staged_operand(model, engines, kv, counts=(1, 4, 5, 8)):
    """test_staged_operand on the engines `engines` returns, with the qkv K split planned for their SM count, for the
    utterance counts `counts` (path C must take each)."""
    e = engines("bf16", kv, "BC", MAXU)
    o_g, o_w = e.offsets[5], e.offsets[5 + 1]
    g1 = e.arena[o_g:o_g + 2 * D].view(torch.bfloat16)
    Wqkv = e.arena[o_w:o_w + 2 * 3 * D * D].view(torch.bfloat16).view(3 * D, D)
    gen = torch.Generator(device="cuda").manual_seed(5)
    gain = (1 + 0.1 * torch.randn(D, generator=gen, device="cuda")).to(torch.bfloat16)
    depth = 8 + 5 + 8 + plan_pc(3 * D, D, e.n_sm) + 2
    sp = e.sl("spk", torch.float32).view(MAXU, D).clone()
    worst = 0.0
    sens = {"speaker dropped": [], "other row's token": [], "position row pos + 1": []}
    try:
        g1.copy_(gain)
        Wqkv[D:2 * D] = torch.eye(D, device="cuda").to(torch.bfloat16)
        torch.cuda.synchronize()
        for n in counts:
            e.m._kv.zero_()
            tc, tu, ps = design(n, 100 + n)
            begin(e, n, tc, tu, ps)
            x = step_x(e, n, "C", "c_x")
            toks, poss, slots, cond = body_rows(n, tc, tu, ps)
            assert torch.equal(x, x_rows(model, sp, toks, poss, slots, cond)), f"kv {kv} n={n}: x of the owner CTA"
            k = torch.stack([e.cache[0, 0, r, :, poss[r]].reshape(D) for r in range(2 * n)]).double()

            def ref(xx):
                nh, _, s = operand(xx.double(), gain, "C")
                y, A = nh * s, nh.abs() * s
                b = lin_bound("C", "qkv", y, A, e.n_sm) + tau_ss(depth) * A
                if kv == "bf16":
                    b = b + BF16_U * (y.abs() + b)
                return y, b
            y, b = ref(x)
            worst = max(worst, check_bound(f"staged operand kv {kv} n={n}", k, y, b))
            c = torch.tensor(cond, device="cuda")
            swap = [toks[r ^ 1] for r in range(2 * n)]
            pnext = [p + 1 if p + 1 < BLOCK else p - 1 for p in poss]
            for name, xa, rows in (("speaker dropped", x_rows(model, sp, toks, poss, slots, [False] * (2 * n)), c),
                                   ("other row's token", x_rows(model, sp, swap, poss, slots, cond), torch.ones_like(c)),
                                   ("position row pos + 1", x_rows(model, sp, toks, pnext, slots, cond), torch.ones_like(c))):
                sens[name].append(over(k, ref(xa)[0], b)[rows])
    finally:
        g1.fill_(1.0)
        Wqkv.zero_()
        torch.cuda.synchronize()
    for name, v in sens.items():
        caught(f"staged operand kv {kv}: {name}", float(torch.cat([t.flatten() for t in v]).double().mean()), BOUND_SENS)
    print(f"staged layer-0 operand, path C kv {kv}, n_utts {list(counts)}, {e.n_sm} SMs: max |err|/bound {worst:.2e}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. prefill plumbing
def prefill_idx(S, seed):
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, V, (2, S), generator=g, dtype=torch.int32)
    idx[1] = (idx[0] + 1 + torch.randint(0, V - 1, (S,), generator=g, dtype=torch.int32)) % V
    for j, t in enumerate(TOK_EDGE):
        if j < S:
            idx[0, S - 1 - j] = t
    return idx


def chunk_launches(fmt, S, all_pos):
    """launches of one mvb_s1_forward on the 64-token chunk path (module docstring)."""
    n_chunks = -(-S // 64)
    per = 1 + 1 + NL * (9 + (fmt != "bf16")) + (2 if all_pos else 0)
    return n_chunks * per + 4


def forward(e, utt, idx, pos0, all_pos):
    from mvb200 import _lib
    S = idx.shape[1]
    G = 2 * V
    n = 2 * S * V if all_pos else 2 * V
    buf = torch.full((n + 2 * G,), float("nan"), device="cuda")
    d_idx = idx.cuda().contiguous()
    n0 = e.launches()
    _lib.check(e.lib.mvb_s1_forward(e.h, utt, d_idx.data_ptr(), S, pos0, buf[G:].data_ptr(), int(all_pos), e.st()))
    torch.cuda.synchronize()
    nl = e.launches() - n0
    assert torch.isnan(buf[:G]).all() and torch.isnan(buf[G + n:]).all(), f"S={S}: writes outside the caller's buffer"
    out = buf[G:G + n]
    assert not torch.isnan(out).any(), f"S={S} all_positions={all_pos}: elements of the caller's buffer left unwritten"
    return out.view(2, S, V) if all_pos else out.view(2, V), nl


def head_ref(e, x, body):
    """float64 logits [R, V] and bound of the head over x [R, D] (float32) as body `body` stages it.  The fp8 engine's
    path A head is k_gemv_f8: the gamma of tests/test_fp8_gemv_gpu.py (hi + lo activation terms, RMSNorm) and its sum of
    squares (a lane's D / 32-term fma chain, 2 shuffles, 8 warp sums, / D, + eps: depth D / 32 + 12)."""
    W, s = e.weights("lm_heads.0.weight", V, D)
    nh, _, rs = operand(x.double(), e.model.gf, body)
    sc = 1.0 if s is None else s[None, :]
    y = (nh @ W.t()) * rs * sc
    A = (nh.abs() @ W.abs().t()) * rs * sc
    if e.fmt == "fp8" and body == "A":
        from test_fp8_gemv_gpu import gamma as gamma_f8
        b = (gamma_f8(D, True) + tau_ss(D // 32 + 12)) * A
    else:
        b = lin_bound(body, "head", y, A, e.n_sm) + tau_ss(SS_DEPTH_AB) * A
    if s is not None:
        b = b + U * y.abs()
    return y, b


def run_prefill(e, utt, S, pos0, seed, sens=None):
    """One prefill case with all_positions = 1 and = 0; returns the worst |err|/bound."""
    model = e.model
    body = "B" if (S >= 2 and "B" in e.tc) else "A"
    idx = prefill_idx(S, seed)
    lgw = e.sl("logits", torch.float32).view(2 * e.utts, V)
    spk = e.sl("spk", torch.float32).view(e.utts, D)
    sp = spk.clone()
    state = {k: e.sl(k, torch.int32).clone() for k in ("slot_map", "pos", "row_tok")}
    gen = torch.Generator(device="cuda").manual_seed(seed)
    lgw.copy_(torch.randn(lgw.shape, generator=gen, device="cuda"))
    lg_before = lgw.clone()
    before = e.before
    others = torch.arange(2 * e.utts, device="cuda") // 2 != utt
    worst = 0.0
    got_last = None
    for all_pos in (True, False):
        out, nl = forward(e, utt, idx, pos0, all_pos)
        want_nl = chunk_launches(e.fmt, S, all_pos) if body == "B" else S * (1 + LAUNCHES["A"] - 1)
        assert nl == want_nl, f"{e.fmt} S={S}: {nl} launches, the {body} prefill path takes {want_nl}"
        # KV cache: the slot's two rows at [pos0, pos0 + S) hold the zero k, v; everything else is as before
        win = e.cache[:, :, 2 * utt:2 * utt + 2, :, pos0:pos0 + S]
        assert (win == 0).all(), f"{e.fmt} S={S}: appended k / v of the zero layers are not 0"
        win.copy_(before[:, :, 2 * utt:2 * utt + 2, :, pos0:pos0 + S])
        assert torch.equal(e.cache.view(torch.uint8), before.view(torch.uint8)), \
            f"{e.fmt} slot {utt} S={S} pos0={pos0}: KV-cache entries outside the prefill window changed"
        assert torch.equal(lgw[others], lg_before[others]), f"{e.fmt} slot {utt}: other slots' logits rows changed"
        assert torch.equal(spk, sp), f"{e.fmt} slot {utt}: spk entries changed"
        st = {k: e.sl(k, torch.int32) for k in state}
        assert int(st["slot_map"][0]) == utt and torch.equal(st["slot_map"][1:], state["slot_map"][1:])
        want_pos = state["pos"].clone()
        want_pos[utt] = pos0 + S - 1
        assert torch.equal(st["pos"], want_pos), f"{e.fmt} slot {utt} S={S}: decode positions"
        want_rt = state["row_tok"].clone()
        want_rt[2 * utt:2 * utt + 2] = idx[:, S - 1].cuda()
        assert torch.equal(st["row_tok"], want_rt), f"{e.fmt} slot {utt} S={S}: row_tok"
        if body == "B":
            s0 = (S - 1) // 64 * 64
            Sc = S - s0
            rw = e.sl("b_rows", torch.int32).view(5, 128)[:, :2 * Sc].cpu()
            c = torch.arange(2 * Sc) // Sc
            s = torch.arange(2 * Sc) % Sc
            want = torch.stack([2 * utt + c, pos0 + s0 + s, idx[c, s0 + s].long(), torch.full_like(c, utt), (c == 0).long()])
            assert torch.equal(rw.long(), want), f"{e.fmt} S={S}: row map of the last chunk"
        if all_pos:
            s_all = torch.arange(S)
            toks = torch.cat([idx[0], idx[1]]).tolist()
            poss = (pos0 + torch.cat([s_all, s_all])).tolist()
            cond = [True] * S + [False] * S
            x = x_rows(model, sp, toks, poss, [utt] * (2 * S), cond)
            y, b = head_ref(e, x, body)
            got = out.reshape(2 * S, V).double()
            worst = max(worst, check_bound(f"{e.fmt}/{e.kv} slot {utt} S={S} pos0={pos0} logits", got, y, b))
            last = torch.tensor([S - 1, 2 * S - 1])
            yl, bl = y[last], b[last]
            if sens is not None:
                alt = {}
                if pos0 > 0:
                    alt["position row pos0 + s0 + s - 1"] = (x_rows(model, sp, toks, [p - 1 for p in poss], [utt] * (2 * S), cond), None)
                if S > 64:
                    tt = torch.cat([idx[0, s_all % 64], idx[1, s_all % 64]]).tolist()
                    alt["chunk offset s0 dropped from the token index"] = (x_rows(model, sp, tt, poss, [utt] * (2 * S), cond),
                                                                          torch.cat([s_all, s_all]) >= 64)
                alt["uncond tokens from row 0"] = (x_rows(model, sp, idx[0].tolist() * 2, poss, [utt] * (2 * S), cond),
                                                   torch.tensor([False] * S + [True] * S))
                alt["slot u - 1's speaker"] = (x_rows(model, sp, toks, poss, [utt] * (2 * S), cond, spk_shift=1),
                                               torch.tensor(cond))
                alt["speaker on both rows"] = (x_rows(model, sp, toks, poss, [utt] * (2 * S), cond, spk_both=True),
                                               torch.tensor([False] * S + [True] * S))
                for name, (xa, rows) in alt.items():
                    o = over(got, head_ref(e, xa, body)[0], b)
                    if rows is not None:
                        o = o[rows.cuda()]
                    sens.setdefault(name, []).append(o.flatten())
                if S >= 2:
                    sens.setdefault("last-position gather from row Sc - 2", []).append(
                        over(lgw[2 * utt:2 * utt + 2].double(), y[last - 1], bl).flatten())
        else:
            got_last = out.double()
        # the sampler rows: the last position through the R = 2 head (all_positions = 0: equal to the caller's copy)
        rows = lgw[2 * utt:2 * utt + 2].double()
        worst = max(worst, check_bound(f"{e.fmt}/{e.kv} slot {utt} S={S} pos0={pos0} sampler rows", rows, yl, bl))
    assert torch.equal(got_last, lgw[2 * utt:2 * utt + 2].double()), "the 2 x V copy differs from the sampler rows"
    return worst


PREFILL_ENGINES = [("bf16", "bf16"), ("bf16", "fp32"), ("int8", "fp32"), ("int8", "bf16"), ("int4", "bf16"), ("int4", "fp32"),
                   ("fp8", "fp32"), ("fp8", "bf16")]


@pytest.mark.parametrize("fmt,kv", PREFILL_ENGINES, ids=[f"{f}-{k}" for f, k in PREFILL_ENGINES])
def test_prefill(model, engines, fmt, kv):
    prefill_cases(engines, fmt, kv, PREFILL)


def prefill_cases(engines, fmt, kv, cases):
    """test_prefill for the (S, pos0) cases on the engines `engines` returns (their SM count may be capped)."""
    e = engines(fmt, kv, "BC", MAXU)
    gen = torch.Generator(device="cuda").manual_seed(3)
    e.m._kv.view(e.dt).copy_(torch.randn(e.m._kv.numel() // e.cache.element_size(), generator=gen, device="cuda"))
    e.before = e.cache.clone()
    worst = 0.0
    sens = {}
    try:
        for utt in (0, MAXU - 1):
            for i, (S, pos0) in enumerate(cases):
                sens_case = sens if (utt == MAXU - 1 and (S, pos0) in ((70, 1000), (129, 0))) else None
                worst = max(worst, run_prefill(e, utt, S, pos0, 1000 * utt + i, sens_case))
    finally:
        e.before = None
    for name, v in sens.items():
        caught(f"prefill {fmt}/{kv}: {name}", float(torch.cat(v).double().mean()), BOUND_SENS)
    print(f"prefill {fmt} engine, kv {kv}, {e.n_sm} SMs: {len(cases)} cases x slots 0, {MAXU - 1}: max |err|/bound {worst:.2e}; "
          f"peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def test_prefill_path_a(model, engines):
    """tensor_core_path = "": the one-position path A loop at every length."""
    prefill_path_a(engines, "bf16")


def test_prefill_path_a_fp8(model, engines):
    """The path A loop of an fp8 engine: k_gemv_f8 for every projection, the head with the bound of k_gemv_f8."""
    prefill_path_a(engines, "fp8")


def prefill_path_a(engines, fmt):
    e = engines(fmt, "fp32", "", 3)
    e.m._kv.zero_()
    e.before = e.cache.clone()
    worst = 0.0
    try:
        for i, (utt, S, pos0) in enumerate([(0, 2, 0), (2, 65, 1977)]):
            worst = max(worst, run_prefill(e, utt, S, pos0, 77 + i))
    finally:
        e.before = None
    print(f"prefill {fmt}, path A loop (S = 2, 65): max |err|/bound {worst:.2e}")
