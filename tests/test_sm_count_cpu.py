"""CPU: the SM-count test hook's argument checks, and the host-planning mirrors that tests/test_sm_count_gpu.py uses to
predict what the stage-1 engine plans on a part with G SMs (the H100 SXM has 132, the H100 PCIe 114, the H20 78, a MIG
slice fewer):
  plan_pc       the K split S of each persistent-kernel phase (test_decode_linear_ops_gpu.plan_pc);
  att_fits      pc_att_fits: the per-CTA attention tile table (<= 128 tiles) and split count (<= 64);
  owner_ok      CTA 2 (n_utts - 1), the only CTA that writes the last batch entry's x rows and decode state back, exists;
  fused_ok      the grid sampler gives each CTA ceil(V / G) <= 32 vocabulary entries;
  body          which decode body mvb_s1_decode runs: "C-fused", "C" (persistent kernel + k_sample), "B" or "A".
The values checked here are derived by hand from the formulas, not read back from the mirrors."""
import ctypes

import pytest

from test_decode_linear_ops_gpu import plan_pc

PC_RPAD, PC_MAX_TILES, PC_MAX_CHUNKS, PC_SAMP_OWN, SAMP_PAD = 16, 128, 64, 32, 4096
SM_COUNTS = [132, 131, 114, 97, 81, 80, 78, 64, 60, 32, 16, 8]
TINY_SM_COUNTS = [1, 2, 3, 7]
# (dim, n_head, intermediate, vocab) of the production stage-1 model and of synth.TINY
FULL = (2048, 16, 5632, 2562)
TINY = (256, 2, 768, 2562)


def phases(dims):
    """(M, K) of the five persistent-kernel phases: qkv, wo, w1|w3, w2, head."""
    D, _, F, V = dims
    return [(3 * D, D), (D, D), (2 * F, D), (D, F), (V, D)]


def pc_ok(dims, G, kv, block):
    """Mirror of create_engine's pc_ok for a production-architecture bf16 engine with a checkpoint-ordered arena."""
    D, _, F, _ = dims
    kv_ok = kv == "fp32" or block % 64 == 0
    staging_ok = F * 8 <= 48 * 1024 - 256
    return kv_ok and staging_ok and F % 128 == 0 and D % 128 == 0 and all(plan_pc(M, K, G) > 0 for M, K in phases(dims))


def att_tiles(G, n_utts, H, kv, block):
    """(Z, tiles of the busiest CTA) of pc_att_fits's bound."""
    R, ppc = 2 * n_utts, 32 if kv == "fp32" else 64
    TT = -(-block // ppc)
    Z = min(max(1, G // (R * H)), TT)
    return Z, -(-R * H * Z // G) * -(-TT // Z)


def att_fits(G, n_utts, H, kv, block):
    Z, tiles = att_tiles(G, n_utts, H, kv, block)
    return Z <= PC_MAX_CHUNKS and tiles <= PC_MAX_TILES


def owner_ok(G, n_utts):
    return 2 * n_utts - 1 <= G


def fused_ok(G, V):
    return -(-V // G) <= PC_SAMP_OWN and V <= SAMP_PAD


def path_c(dims, G, n_utts, kv, block):
    """Mirror of use_path_c."""
    return (pc_ok(dims, G, kv, block) and 2 * n_utts <= PC_RPAD and owner_ok(G, n_utts)
            and att_fits(G, n_utts, dims[1], kv, block))


def body(dims, G, n_utts, kv, block):
    """The body mvb_s1_decode runs for n_utts utterances with top_k = 0, no guidance link and the fused sampler enabled."""
    if path_c(dims, G, n_utts, kv, block):
        return "C-fused" if fused_ok(G, dims[3]) else "C"
    return "B" if n_utts >= 2 else "A"


# ---------------------------------------------------------------------------------------------------------------------
def test_sm_limit_argument_checks():
    """n < 0 is rejected with MVB_ERR_ARG and a message naming the hook; n = 0 and n > 0 are accepted.  No GPU is
    touched: the limit lives in the library."""
    from mvb200 import _lib
    lib = _lib.load()
    try:
        for bad in (-1, -132, -2 ** 31):
            assert lib.mvb_test_set_sm_limit(bad) == _lib.MVB_ERR_ARG, bad
            assert b"mvb_test_set_sm_limit" in lib.mvb_last_error()
        for ok in (0, 1, 114, 132, 10 ** 6, 0):
            assert lib.mvb_test_set_sm_limit(ok) == _lib.MVB_OK, ok
    finally:
        assert lib.mvb_test_set_sm_limit(0) == _lib.MVB_OK
    assert isinstance(lib.mvb_test_set_sm_limit.argtypes[0](0), ctypes.c_int32)


# S and KB = K / 64 of each phase at 132 and 114 SMs (production width): "even" when S divides KB
PLAN_TABLE = {
    132: {"qkv": (8, 32), "wo": (16, 32), "w13": (6, 32), "w2": (22, 88), "head": (11, 32)},
    114: {"qkv": (7, 32), "wo": (11, 32), "w13": (5, 32), "w2": (18, 88), "head": (16, 32)},
}


@pytest.mark.parametrize("G", list(PLAN_TABLE))
def test_plan_pc_mirror_table(G):
    got = {name: (plan_pc(M, K, G), K // 64) for name, (M, K) in zip(PLAN_TABLE[G], phases(FULL))}
    assert got == PLAN_TABLE[G]
    even = {name: KB % S == 0 for name, (S, KB) in got.items()}
    # at 132 SMs qkv, wo and w2 split K evenly; at 114 only the head does
    assert even == ({"qkv": True, "wo": True, "w13": False, "w2": True, "head": False} if G == 132 else
                    {"qkv": False, "wo": False, "w13": False, "w2": False, "head": True})


def test_plan_pc_mirror_declines_too_few_ctas():
    """A CTA stages at most 12 k-blocks per phase: at production width w2 (K = 5632, 88 k-blocks) needs S >= 8, so fewer
    than 8 SMs cannot run path C there; the tiny model's K = 256 / 768 fit one CTA."""
    assert plan_pc(2048, 5632, 7) == 0 and plan_pc(2048, 5632, 8) == 8
    assert plan_pc(3 * 2048, 2048, 2) == 0 and plan_pc(3 * 2048, 2048, 3) == 3
    assert not pc_ok(FULL, 7, "fp32", 2048) and pc_ok(FULL, 8, "fp32", 2048)
    assert all(pc_ok(TINY, G, "bf16", 2048) for G in TINY_SM_COUNTS)


def test_fused_sampler_slots():
    """V = 2562: a CTA owns ceil(V / G) entries, 8 slots per compute warp.  At 132 it owns 20 (slots t = 5 .. 7 never
    hold an entry), at 114 23, at 81 all 32; at 80 it would need 33 and the host declines the fused sampler."""
    V = 2562
    assert [-(-V // G) for G in (132, 131, 114, 81, 80)] == [20, 20, 23, 32, 33]
    assert [fused_ok(G, V) for G in (132, 131, 114, 81, 80, 78)] == [True, True, True, True, False, False]
    assert fused_ok(128, 4096) and fused_ok(131, 4096) and not fused_ok(127, 4096)


# (G, n_utts, kv) at which the busiest CTA owns exactly PC_MAX_TILES tiles at block_size 2048, H = 16
CAPACITY_EDGES = [(132, 8, "fp32"), (16, 1, "fp32"), (64, 4, "fp32"), (64, 8, "bf16"), (8, 1, "bf16")]


@pytest.mark.parametrize("G,n,kv", CAPACITY_EDGES)
def test_attention_capacity_edges(G, n, kv):
    TT = 64 if kv == "fp32" else 32
    assert att_tiles(G, n, 16, kv, 2048) == (1, -(-32 * n // G) * TT) == (1, 128)
    assert att_fits(G, n, 16, kv, 2048)
    # fewer SMs: over the table (8 fp32 utterances hold 2 units of 64 tiles per CTA down to 128 SMs)
    assert not att_fits(127 if G == 132 else G - 1, n, 16, kv, 2048)
    if n < 8:
        assert not att_fits(G, n + 1, 16, kv, 2048)      # one utterance more: over the table


def test_owner_guard_examples():
    """Batches whose tile table fits although CTA 2 (n_utts - 1) does not exist: the guard sends them to path B."""
    # production width, block_size 256, bf16 cache (the probe engine of test_decode_linear_ops_gpu.py), 8 utterances
    for G in range(8, 15):
        assert pc_ok(FULL, G, "bf16", 256) and att_fits(G, 8, 16, "bf16", 256), G
        assert not owner_ok(G, 8) and body(FULL, G, 8, "bf16", 256) == "B", G
    assert owner_ok(15, 8) and body(FULL, 15, 8, "bf16", 256) == "C"
    # the tiny model, bf16 cache, 2 utterances on 2 SMs: 4 units of 32 tiles per CTA fit exactly
    assert att_tiles(2, 2, 2, "bf16", 2048) == (1, 128) and pc_ok(TINY, 2, "bf16", 2048)
    assert not owner_ok(2, 2) and body(TINY, 2, 2, "bf16", 2048) == "B"
    assert body(TINY, 3, 2, "bf16", 2048) == "C"
    # at 132 SMs the guard never binds: 2 n - 1 <= 15
    assert all(owner_ok(132, n) for n in range(1, 9))


def test_body_mirror_at_132_matches_the_existing_modules():
    """At 132 SMs the mirror gives what the existing op-level modules assert: the fused persistent kernel for 1 .. 8
    utterances at production width, block_size 256 and 2048, either cache; 114 SMs already send 8 fp32 utterances at
    block_size 2048 to path B."""
    for kv in ("fp32", "bf16"):
        assert all(body(FULL, 132, n, kv, 256) == "C-fused" for n in range(1, 9))
        assert all(body(FULL, 132, n, kv, 2048) == "C-fused" for n in range(1, 9))
    assert body(FULL, 114, 8, "fp32", 2048) == "B"        # 8 fp32 utterances exceed the table below 132 SMs
