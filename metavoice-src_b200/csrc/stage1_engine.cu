// libmvb200: host side of the stage-1 engine and its C ABI (include/mvb200.h).
// No torch, no CPU fallback: every entry point either runs the CUDA path or fails loudly.
#include <cuda_runtime.h>

#include <cmath>
#include <algorithm>
#include <cstring>
#include <deque>
#include <map>
#include <vector>

#include "host.cuh"
#include "stage1_kernels.cuh"
#include "tc_gemm_host.cuh"
#include "decode_persistent.cuh"
#include "gemv_w4.cuh"
#include "gemv_w8.cuh"
#include "gemv_f8.cuh"

using namespace mvb;

struct WsLayout {
  size_t x, qkv, att, ffn, logits, spk, part_o, part_ml;
  size_t slot_map, pos, row_tok, done, n_gen, gen_tokens, sampled, samp, noise, forced, ticket, budget, noise_base;
  size_t stage_idx, stage_spk, stage_forced, stage_noise;
  // path B (tensor-core rows path): activations for up to RB_MAX rows
  size_t b_x, b_qkv, b_att, b_ffn, b_logits, b_last, b_B, b_rows, b_scratch, b_tickets, b_part_o, b_part_ml, b_att_tickets;
  // path C (persistent decode kernel)
  size_t c_x, c_qkv, c_gu, c_part_o, c_part_ml, c_bar, c_trace, c_stat, c_samp_part, c_samp_best;
  size_t total;
  // an int4, int8 or fp8 engine's workspace continues with the one-layer bf16 weight scratch; an int8 or fp8 engine's
  // then with lm_head's widened q; an fp8 engine's then with speaker_cond_pos's widened q
  size_t layer_scratch, total_int4, w8_head, total_int8, f8_spk, total_fp8;
};

constexpr int RB_MAX = 128;        // rows per tensor-core pass: 64-token prefill chunk x 2 CFG rows, or 64 utterances
constexpr int PREFILL_CHUNK = 64;
constexpr int GEN_BURST = 32;       // decode steps between two host polls of the done flags in mvb_s1_generate

// elements of one layer's bf16 weight scratch: wqkv, wo, w1, w3, w2
static size_t layer_scratch_elems(const mvb_s1_config& c) {
  const size_t D = c.dim, F = c.intermediate;
  return 4 * D * D + 3 * D * F;
}

// Storage format of the Linear weights of an engine's arena (include/mvb200.h): bf16 (mvb_s1_create), int4 packed
// matrices for the five layer matrices (mvb_s1_create_int4), int8 matrices for every Linear (mvb_s1_create_int8), fp8
// matrices for every Linear (mvb_s1_create_fp8).
enum class WFmt { BF16, INT4, INT8, FP8 };

struct Mk { int M, K; };
// [M, K] of layer tensor t (1 wqkv, 2 wo, 4 w1, 5 w3, 6 w2; {0, 0} for the norms)
static Mk layer_mk(const mvb_s1_config& c, int t) {
  const int D = c.dim, F = c.intermediate;
  const Mk mk[7] = {{0, 0}, {3 * D, D}, {D, D}, {0, 0}, {F, D}, {F, D}, {D, F}};
  return mk[t];
}

static WsLayout make_layout(const mvb_s1_config& c) {
  WsLayout L;
  const size_t U = c.max_utts, R = 2 * U, D = c.dim, F = c.intermediate, V = c.vocab, H = c.n_head;
  WsBump ws;
  L.x = ws.take(R * D * 4);
  L.qkv = ws.take(R * 3 * D * 4);
  L.att = ws.take(R * D * 4);
  L.ffn = ws.take(R * F * 4);
  L.logits = ws.take(R * V * 4);
  L.spk = ws.take(U * D * 4);
  L.part_o = ws.take(R * H * ATT_SPLITS * 128 * 4);
  L.part_ml = ws.take(R * H * ATT_SPLITS * 2 * 4);
  L.slot_map = ws.take(U * 4);
  L.pos = ws.take(U * 4);
  L.row_tok = ws.take(R * 4);
  L.done = ws.take(U * 4);
  L.n_gen = ws.take(U * 4);
  L.gen_tokens = ws.take(U * (size_t)c.max_new * 4);
  L.sampled = ws.take(U * (size_t)c.max_new * 4);
  L.samp = ws.take(U * sizeof(SamplingDev));
  L.noise = ws.take(U * sizeof(void*));
  L.forced = ws.take(U * sizeof(void*));
  L.ticket = ws.take(R * H * 4);
  L.budget = ws.take(U * 4);
  L.noise_base = ws.take(U * 4);
  L.stage_idx = ws.take(U * 2 * (size_t)c.block_size * 4);
  L.stage_spk = ws.take(U * (size_t)c.spk_dim * 4);
  L.stage_forced = ws.take(U * (size_t)c.max_new * 4);
  L.stage_noise = ws.take(U * (size_t)GEN_BURST * V * 4);   // host-supplied Exp(1) draws are staged one burst at a time
  {
    const size_t RB = RB_MAX, NBM = 2 * RB_MAX;
    L.b_x = ws.take(RB * D * 4);
    L.b_qkv = ws.take(RB * 3 * D * 4);
    L.b_att = ws.take(RB * D * 4);
    L.b_ffn = ws.take(RB * F * 4);
    L.b_logits = ws.take(RB * V * 4);
    L.b_last = ws.take(2 * D * 4);
    L.b_B = ws.take(NBM * (F > D ? F : D) * 2);
    L.b_rows = ws.take(5 * RB * 4);
    size_t sc = 0;
    const size_t mats[5][3] = {{3 * D, D, 1}, {D, D, 1}, {F, D, 2}, {D, F, 1}, {V, D, 1}};
    for (auto& m : mats) {
      GemmPlan g = plan_gemm((int)m[0], (int)m[1], (int)NBM, m[2] == 2, GEMM_MAX_SM);
      if (g.scratch_floats > sc) sc = g.scratch_floats;
    }
    L.b_scratch = ws.take(sc * 4);
    L.b_tickets = ws.take(256 * 4);
    L.b_part_o = ws.take(RB * H * ATT_SPLITS * 128 * 4);
    L.b_part_ml = ws.take(RB * H * ATT_SPLITS * 2 * 4);
    L.b_att_tickets = ws.take(RB * H * 4);
  }
  L.c_x = ws.take((size_t)PC_RPAD * D * 4);
  L.c_qkv = ws.take((size_t)PC_RPAD * 3 * D * 4);
  L.c_gu = ws.take((size_t)PC_RPAD * 2 * F * 4);
  L.c_part_o = ws.take((size_t)PC_RPAD * H * PC_MAX_CHUNKS * 128 * 4);
  L.c_part_ml = ws.take((size_t)PC_RPAD * H * PC_MAX_CHUNKS * 2 * 4);
  L.c_bar = ws.take(256);
  L.c_trace = ws.take((size_t)160 * PC_TRACE_EVENTS * 8);
  L.c_stat = ws.take((size_t)(2 * c.n_layer + 1) * PC_RPAD * 4);
  L.c_samp_part = ws.take((size_t)(PC_RPAD / 2) * 256 * 4);
  L.c_samp_best = ws.take((size_t)2 * (PC_RPAD / 2) * 8);
  L.total = ws.end;
  L.layer_scratch = ws.take(layer_scratch_elems(c) * 2);
  L.total_int4 = ws.end;
  L.w8_head = ws.take((size_t)c.vocab * c.dim * 2);
  L.total_int8 = ws.end;
  L.f8_spk = ws.take((size_t)c.dim * c.spk_dim * 2);
  L.total_fp8 = ws.end;
  return L;
}

// Per-layer norm parameters and Linear biases, null where the architecture has none (the production one: every beta and
// bias).
struct S1LayerP {
  const __nv_bfloat16 *g1, *b1, *g2, *b2;                   // ln_1 / ln_2 gain and (LayerNorm with bias) beta
  const __nv_bfloat16 *qkv_b, *o_b, *fc_b, *fc3_b, *proj_b;  // c_attn, attn.c_proj, c_fc | w1, w3, mlp.c_proj
};

// A voice (mvb_s1_add_voice): the tensors of layers [first_layer, n_layer) and ln_f in an overlay; every other tensor is
// the base checkpoint's.  Voice 0, the base, has first_layer = n_layer + 1, so that it uses the base ln_f too.
struct S1Voice {
  int first_layer = 0;
  std::vector<const __nv_bfloat16*> t;   // 7 per overlaid layer, indexed like mvb_s1::lw's t (GELU: 5 unused)
  std::vector<S1LayerP> lp;              // per overlaid layer
  std::vector<CUtensorMap> tmW;          // 5 per overlaid layer, as mvb_s1::tmW
  const __nv_bfloat16 *lnf_g = nullptr, *lnf_b = nullptr;
};

// The voice grouping of one batch of decode entries: groups in order of descending first_layer (voice 0 first), each
// group's entries in batch order.  At any layer the groups still on the base weights are then a prefix of the order.
struct VoicePlan {
  int n = 0;                                    // groups
  int voice[MVB_S1_MAX_VOICES];
  int start[MVB_S1_MAX_VOICES + 1];             // group g = order[start[g] .. start[g + 1])
  int grp[64];                                  // voice group of every batch entry
};
// Batch entries in group order, by value into k_voice_slots (captured into the step graph).
struct VoiceOrder {
  int entry[64];
  int n;
};
// vslots[i] = slot_map[order.entry[i]]: the slot map of the grouped order, whose slices are the voice groups.
__global__ void k_voice_slots(const int* __restrict__ slot_map, VoiceOrder order, int* __restrict__ vslots) {
  const int i = threadIdx.x;
  if (i < order.n) vslots[i] = slot_map[order.entry[i]];
}
// Path B with voice groups: row_grp[r] = voice group of decode row r (batch entry r / 2), for k_tc_gemm_grp.
struct VoiceRows {
  int grp[64];
};
__global__ void k_voice_rows(VoiceRows v, int R, int* __restrict__ row_grp) {
  const int r = threadIdx.x;
  if (r < R) row_grp[r] = v.grp[r >> 1];
}

// Step graphs keyed by a voice grouping are cached up to this many, oldest evicted first (see run_body).
constexpr int VOICE_GRAPHS_MAX = 32;

struct mvb_s1 {
  mvb_s1_config cfg;
  mvb_s1_arch arch{};                                 // all zero: the production architecture (rmsnorm, swiglu, no bias)
  std::vector<S1LayerP> lp;
  const __nv_bfloat16* lnf_b = nullptr;               // ln_f beta (LayerNorm with bias)
  int n_sm = 132;
  const char* arena = nullptr;
  std::vector<uint64_t> off;
  char* kv = nullptr;
  char* ws = nullptr;
  WsLayout L;
  S1State st;
  std::map<int, cudaGraphExec_t> graphs;
  cudaStream_t cap_stream = nullptr;
  uint64_t launches = 0;
  std::map<int, int> graph_nodes;
  int* h_flags = nullptr;  // pinned: done flags / counters read back by generate()
  // path B
  std::vector<CUtensorMap> tmW;                       // per layer {wqkv, wo, w1, w3, w2}, then lm_head
  std::map<std::pair<int, int>, CUtensorMap> tmB;     // (NB, K) -> activation buffer map
  bool path_b = true;                                 // tensor-core rows path for batched decode and prefill
  RowsDev rows;
  // path C
  bool path_c = true;
  bool pc_ok = false;
  bool trace = false;
  bool fused = true;                                  // sample inside the persistent kernel (multi-token launches)
  CUtensorMap tm_kv;                                  // bf16 cache: 2-D map over the whole KV arena: [rows = layer, k|v, cache row, head, pos][128]
  CUtensorMap tm3[6];                                 // 3-D (k, row, layer) maps: wqkv, wo, w1, w3, w2, head
  PcMat pm[5];
  std::vector<int> h_topk;                            // top_k of every utterance slot as installed by mvb_s1_begin
  std::vector<int> h_link;                            // SamplingDev::link of every slot as installed by mvb_s1_admit_guided
  size_t layer_stride_elems = 0;
  // voices: [0] is the base; next_voice is what mvb_s1_set_voice selected, slot_voice what the slot was admitted with
  std::vector<S1Voice> voices;
  std::vector<int> next_voice, slot_voice;
  // device buffers of the first mvb_s1_add_voice: [64] k_voice_slots' grouped slot map, then [RB_MAX] k_voice_rows'
  // row groups; split-K counters of the grouped GEMM; every voice's path-B tensor maps (voice_tm)
  int* vslots = nullptr;
  int* row_grp = nullptr;
  unsigned* vtickets = nullptr;
  CUtensorMap* d_tm = nullptr;
  std::map<std::vector<int>, cudaGraphExec_t> vgraphs;   // {use_b, n_utts, voice of every entry} -> step graph
  std::map<std::vector<int>, int> vgraph_nodes;
  std::map<std::vector<int>, cudaEvent_t> vgraph_done;   // recorded after each launch of the graph
  std::deque<std::vector<int>> vgraph_age;            // insertion order of vgraphs' keys
  // int4 engine: wqkv / wo / w1 / w3 / w2 are packed matrices, lm_head stays bf16 (head_fmt).  int8 / fp8 engine: every
  // Linear is an int8 / fp8 matrix.  Path A streams them through k_gemv_w4 / k_gemv_w8 / k_gemv_f8 (launch_gemv; the fp8
  // GEMV serves up to F8_MAX_UTTS slots at once); path B widens one layer at a time into layer_scratch (bf16
  // [wqkv | wo | w1 | w3 | w2]) with `widen`, lm_head's q once at create into w8_head and an fp8 engine's
  // speaker_cond_pos q into f8_spk, and k_tc_gemm applies the int8 / fp8 row scales.
  WFmt fmt = WFmt::BF16;
  __nv_bfloat16* layer_scratch = nullptr;
  __nv_bfloat16* w8_head = nullptr;
  __nv_bfloat16* f8_spk = nullptr;
  bool row_scaled() const { return fmt == WFmt::INT8 || fmt == WFmt::FP8; }   // int8 / fp8 matrices with row scales
  WFmt head_fmt() const { return fmt == WFmt::INT4 ? WFmt::BF16 : fmt; }

  template <typename T>
  T* wsp(size_t o) const { return reinterpret_cast<T*>(ws + o); }
  const __nv_bfloat16* w(int i) const { return reinterpret_cast<const __nv_bfloat16*>(arena + off[i]); }
  bool gelu() const { return arch.mlp == MVB_S1_MLP_GELU; }
  bool layer_norm() const { return arch.norm == MVB_S1_NORM_LAYER; }
  bool production_arch() const { return arch.norm == MVB_S1_NORM_RMS && arch.mlp == MVB_S1_MLP_SWIGLU && !arch.bias; }
  // eps of ln_1 / ln_2 / ln_f: LayerNorm's is fixed at 1e-5 (layers/layers.py:17), RMSNorm's is the config's
  float norm_eps() const { return layer_norm() ? 1e-5f : cfg.norm_eps; }
  // arena tensor t of a layer (0 ln_1, 1 wqkv, 2 wo, 3 ln_2, 4 w1 | c_fc, 5 w3, 6 w2 = mlp.c_proj); a GELU layer has six
  // tensors and no w3
  const __nv_bfloat16* lw(int layer, int t) const {
    const bool g = gelu();
    return w(MVB_S1_GLOBAL_TENSORS + layer * (g ? 6 : MVB_S1_LAYER_TENSORS) + (g && t == 6 ? 5 : t));
  }
  // The same for voice v: its overlay's tensor from its first_layer on, the base's below.
  int first_layer(int v) const { return voices[v].first_layer; }
  bool overlaid(int v, int layer) const { return layer >= voices[v].first_layer; }
  const __nv_bfloat16* vlw(int v, int layer, int t) const {
    return overlaid(v, layer) ? voices[v].t[(size_t)(layer - voices[v].first_layer) * 7 + t] : lw(layer, t);
  }
  const S1LayerP& vlp(int v, int layer) const { return overlaid(v, layer) ? voices[v].lp[layer - voices[v].first_layer] : lp[layer]; }
  // tensor map i (0 wqkv, 1 wo, 2 w1, 3 w3, 4 w2) of a layer of voice v; layer n_layer: lm_head (shared by every voice)
  const CUtensorMap* vtm(int v, int layer, int i) const {
    if (layer < cfg.n_layer && overlaid(v, layer)) return &voices[v].tmW[(size_t)(layer - voices[v].first_layer) * 5 + i];
    return &tmW[(size_t)layer * 5 + (layer < cfg.n_layer ? i : 0)];
  }
  // Device copy of vtm(v, layer, i): n_layer * 5 + 1 maps per voice (layer n_layer: lm_head)
  const CUtensorMap* voice_tm(int v, int layer, int i) const {
    return d_tm + (size_t)v * (cfg.n_layer * 5 + 1) + (size_t)layer * 5 + (layer < cfg.n_layer ? i : 0);
  }
  const __nv_bfloat16* lnf_gain(int v) const { return v ? voices[v].lnf_g : w(3); }
  const __nv_bfloat16* lnf_beta(int v) const { return v ? voices[v].lnf_b : lnf_b; }
  // The one weight-source accessor of the tensor-core path: the bf16 matrix t (1 wqkv, 2 wo, 4 w1, 5 w3, 6 w2) of a layer,
  // i.e. the arena tensor, or for an int4 / int8 / fp8 engine its slot in the layer scratch (k_w4_dequant / k_w8_widen /
  // k_f8_widen fill it).
  const __nv_bfloat16* tc_w(int layer, int t) const {
    if (fmt == WFmt::BF16) return lw(layer, t);
    const size_t D = cfg.dim, F = cfg.intermediate;
    const size_t at[7] = {0, 0, 3 * D * D, 0, 4 * D * D, 4 * D * D + F * D, 4 * D * D + 2 * F * D};
    return layer_scratch + at[t];
  }
  // Row scales of the tensor-core path: those of arena tensor i ([M, K]) for an int8 or fp8 engine, else none.
  const __nv_bfloat16* tc_scale(int i, int M, int K) const {
    if (!row_scaled()) return nullptr;
    return reinterpret_cast<const __nv_bfloat16*>(arena + off[i] + w8_scale_offset(M, K));
  }
  const __nv_bfloat16* tc_lscale(int layer, int t) const {
    const Mk mk = layer_mk(cfg, t);
    return tc_scale(MVB_S1_GLOBAL_TENSORS + layer * MVB_S1_LAYER_TENSORS + t, mk.M, mk.K);
  }
  const __nv_bfloat16* head_scale() const { return tc_scale(4, cfg.vocab, cfg.dim); }
  size_t kv_elem() const { return cfg.kv_dtype == MVB_KV_FP32 ? 4 : cfg.kv_dtype == MVB_KV_FP8 ? 1 : 2; }
  // bytes of one layer's K (or V) elements; an fp8 cache's scales follow all the layers' codes
  size_t kv_half_bytes() const {
    return (size_t)2 * cfg.max_utts * cfg.n_head * cfg.block_size * cfg.head_dim * kv_elem();
  }
  bool kv_f8() const { return cfg.kv_dtype == MVB_KV_FP8; }
  // layer l of an fp8 cache (include/mvb200.h): K / V codes, then K / V scales in the region after every layer's codes
  KvF8 kv_f8_layer(int l) const {
    const size_t half = kv_half_bytes(), n_scales = (size_t)2 * cfg.max_utts * cfg.n_head * cfg.block_size;
    __nv_bfloat16* sc = reinterpret_cast<__nv_bfloat16*>(kv + (size_t)cfg.n_layer * 2 * half) + (size_t)l * 2 * n_scales;
    uint8_t* kc = reinterpret_cast<uint8_t*>(kv + (size_t)l * 2 * half);
    return KvF8{kc, kc + half, sc, sc + n_scales};
  }
};


// Static decomposition of one matrix over `ctas` CTAs: the K split that minimises the busiest CTA's modelled phase time.
static PcMat plan_pc(int M, int K, int ctas, int tile_rows) {
  PcMat best{};
  long best_cost = -1;
  const int T = (M + tile_rows - 1) / tile_rows, KB = K / 64;
  for (int S = 1; S <= KB && S <= 32 && S <= ctas; ++S) {
    const int Gp = ctas / S;
    const int tiles_per = (T + Gp - 1) / Gp;
    const int kb_per = (KB + S - 1) / S;
    if (kb_per > PC_BKB_MAX) continue;
    // Cost of a phase in tile-load units: every tile a CTA owns costs its k-blocks plus ~2.5 for the accumulator drain
    // (slot loads + red.add), and staging the activation operand costs ~2 per k-block of the CTA's K slice (one
    // dependent L2 round trip per 256 chunks).
    const long cost = (long)tiles_per * (2 * kb_per + 5) + 4 * kb_per;
    if (best_cost < 0 || cost < best_cost) {
      best_cost = cost;
      best.T = T; best.KB = KB; best.S = S; best.G = Gp;
    }
  }
  if (best_cost < 0) best.S = 0;
  return best;
}

// Largest K of a path-A GEMV: its two staged fp32 activation rows (2 K floats) must fit in the opt-in shared memory of
// two co-resident CTAs.  The int4 and int8 GEMVs, and every kernel of the resident decode kernel's engine, keep the
// default 48 KB (quant_staging_ok, pc_ok).
constexpr size_t GEMV_MAX_SMEM = 96 * 1024;
static bool default_staging_ok(const mvb_s1_config& c) { return (size_t)c.intermediate * 8 <= 48 * 1024 - 256; }

static int validate(const mvb_s1_config* c) {
  if (!c) return set_error(MVB_ERR_ARG, "null config");
  if (c->head_dim != 128) return set_error(MVB_ERR_UNSUPPORTED, "head_dim must be 128 (got %d)", c->head_dim);
  if (c->dim != c->n_head * c->head_dim) return set_error(MVB_ERR_ARG, "dim != n_head*head_dim");
  if (c->dim % 256 || c->intermediate % 256) return set_error(MVB_ERR_UNSUPPORTED, "dim and intermediate must be multiples of 256");
  if (c->vocab % 2 || c->vocab > SAMP_PAD) return set_error(MVB_ERR_UNSUPPORTED, "vocab must be even and <= %d", SAMP_PAD);
  if (c->max_utts < 1 || c->max_utts > 64) return set_error(MVB_ERR_ARG, "max_utts out of range");
  if (c->max_new < 1 || c->max_new > c->block_size) return set_error(MVB_ERR_ARG, "max_new out of range");
  if (c->kv_dtype != MVB_KV_BF16 && c->kv_dtype != MVB_KV_FP32 && c->kv_dtype != MVB_KV_FP8)
    return set_error(MVB_ERR_ARG, "bad kv_dtype");
  if ((size_t)c->intermediate * 8 > GEMV_MAX_SMEM) return set_error(MVB_ERR_UNSUPPORTED, "intermediate too large for the staging buffer");
  const int known = MVB_S1_NO_ROWS_PATH | MVB_S1_NO_RESIDENT | MVB_S1_UNFUSED_SAMPLER | MVB_S1_TRACE;
  if (c->options & ~known) return set_error(MVB_ERR_ARG, "options: undefined bits 0x%x", (unsigned)(c->options & ~known));
  return MVB_OK;
}

extern "C" size_t mvb_s1_kv_bytes(const mvb_s1_config* c) {
  if (validate(c)) return 0;
  const size_t vecs = (size_t)c->n_layer * 2 * (2 * (size_t)c->max_utts) * c->n_head * c->block_size;   // head vectors
  if (c->kv_dtype == MVB_KV_FP8) return vecs * c->head_dim + vecs * 2;   // e4m3 codes, then one bf16 scale per vector
  return vecs * c->head_dim * (c->kv_dtype == MVB_KV_FP32 ? 4 : 2);
}

extern "C" size_t mvb_s1_workspace_bytes(const mvb_s1_config* c) {
  if (validate(c)) return 0;
  return make_layout(*c).total;
}

// The int4 / int8 GEMVs stage their activations in the default 48 KB of shared memory.
static int quant_staging_ok(const mvb_s1_config* c) {
  if (!default_staging_ok(*c)) return set_error(MVB_ERR_UNSUPPORTED, "intermediate too large for the staging buffer");
  return MVB_OK;
}

extern "C" size_t mvb_s1_int4_workspace_bytes(const mvb_s1_config* c) {
  if (validate(c) || quant_staging_ok(c)) return 0;
  return make_layout(*c).total_int4;
}

extern "C" size_t mvb_s1_int8_workspace_bytes(const mvb_s1_config* c) {
  if (validate(c) || quant_staging_ok(c)) return 0;
  return make_layout(*c).total_int8;
}

extern "C" size_t mvb_s1_fp8_workspace_bytes(const mvb_s1_config* c) {
  if (validate(c) || quant_staging_ok(c)) return 0;
  return make_layout(*c).total_fp8;
}

// Tensors in the offset list: the weights (GELU: six per layer), then, with bias, ln_f.bias (LayerNorm) and per layer
// {ln_1.bias (LayerNorm), c_attn.bias, attn.c_proj.bias, ln_2.bias (LayerNorm), w1.bias, w3.bias | c_fc.bias,
// mlp.c_proj.bias}.
static int s1_offset_count(const mvb_s1_config* c, const mvb_s1_arch& a) {
  const bool ln = a.norm == MVB_S1_NORM_LAYER, gelu = a.mlp == MVB_S1_MLP_GELU;
  int n = MVB_S1_GLOBAL_TENSORS + c->n_layer * (gelu ? 6 : MVB_S1_LAYER_TENSORS);
  if (a.bias) n += (ln ? 1 : 0) + c->n_layer * ((ln ? 2 : 0) + 3 + (gelu ? 1 : 2));
  return n;
}

static int s1_validate_arch(const mvb_s1_arch& a) {
  if (a.norm != MVB_S1_NORM_RMS && a.norm != MVB_S1_NORM_LAYER) return set_error(MVB_ERR_ARG, "arch.norm: undefined value %d", a.norm);
  if (a.mlp != MVB_S1_MLP_SWIGLU && a.mlp != MVB_S1_MLP_GELU) return set_error(MVB_ERR_ARG, "arch.mlp: undefined value %d", a.mlp);
  if (a.bias != 0 && a.bias != 1) return set_error(MVB_ERR_ARG, "arch.bias: undefined value %d", a.bias);
  return MVB_OK;
}

// The matrices of m in format fmt (int4 packed, int8 or fp8) -> bf16 operands of the tensor-core GEMM.
static cudaError_t widen(WFmt fmt, const WidenBatch& m, int n_sm, cudaStream_t s) {
  if (fmt == WFmt::INT4) k_w4_dequant<<<4 * n_sm, 256, 0, s>>>(m);
  else if (fmt == WFmt::INT8) k_w8_widen<<<4 * n_sm, 256, 0, s>>>(m);
  else if (fmt == WFmt::FP8) k_f8_widen<<<4 * n_sm, 256, 0, s>>>(m);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

static int create_engine(const mvb_s1_config* cfg, const mvb_s1_arch* arch, const void* d_arena, size_t arena_bytes,
                         const uint64_t* offsets, void* d_kv, void* d_ws, mvb_s1** out, WFmt fmt) {
  if (int e = validate(cfg)) return e;
  if (fmt != WFmt::BF16)
    if (int e = quant_staging_ok(cfg)) return e;
  const mvb_s1_arch a = arch ? *arch : mvb_s1_arch{};
  if (int e = s1_validate_arch(a)) return e;
  if (!offsets) return set_error(MVB_ERR_ARG, "null pointer argument");
  const int n_off = s1_offset_count(cfg, a);
  if (int e = check_offsets(offsets, n_off, arena_bytes, "weight offset")) return e;
  if (!d_arena || !d_kv || !d_ws || !out) return set_error(MVB_ERR_ARG, "null pointer argument");
  int dev = 0, n_sm = 0, major = 0, minor = 0;
  if (int e = current_device(&dev, &n_sm)) return e;
  MVB_CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  MVB_CK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0) return set_error(MVB_ERR_UNSUPPORTED, "libmvb200 is built for sm_90a only; device is sm_%d%d", major, minor);
  Building<mvb_s1> hb(new mvb_s1(), mvb_s1_destroy);
  mvb_s1* h = hb.get();
  h->cfg = *cfg;
  h->arch = a;
  h->n_sm = n_sm;
  h->arena = reinterpret_cast<const char*>(d_arena);
  h->off.assign(offsets, offsets + n_off);
  {
    const bool ln = h->layer_norm(), gelu = h->gelu();
    int nb = s1_offset_count(cfg, mvb_s1_arch{a.norm, a.mlp, 0});    // first bias slot
    auto bias_slot = [&](bool present) { return present && a.bias ? h->w(nb++) : nullptr; };
    h->lnf_b = bias_slot(ln);
    h->lp.resize(cfg->n_layer);
    for (int l = 0; l < cfg->n_layer; ++l) {
      S1LayerP& p = h->lp[l];
      p.g1 = h->lw(l, 0);
      p.g2 = h->lw(l, 3);
      p.b1 = bias_slot(ln);
      p.qkv_b = bias_slot(true);
      p.o_b = bias_slot(true);
      p.b2 = bias_slot(ln);
      p.fc_b = bias_slot(true);
      p.fc3_b = bias_slot(!gelu);
      p.proj_b = bias_slot(true);
    }
  }
  h->kv = reinterpret_cast<char*>(d_kv);
  h->ws = reinterpret_cast<char*>(d_ws);
  h->L = make_layout(*cfg);
  h->fmt = fmt;
  if (fmt != WFmt::BF16) {
    h->layer_scratch = h->wsp<__nv_bfloat16>(h->L.layer_scratch);
    const bool w8 = h->row_scaled();   // int8 and fp8 matrices share one layout (include/mvb200.h)
    const char* kind = fmt == WFmt::INT8 ? "int8" : fmt == WFmt::FP8 ? "fp8" : "int4 packed";
    for (int l = 0; l < cfg->n_layer; ++l)
      for (int t : {1, 2, 4, 5, 6}) {
        const uint64_t o = h->off[MVB_S1_GLOBAL_TENSORS + l * MVB_S1_LAYER_TENSORS + t];
        const Mk mk = layer_mk(*cfg, t);
        if (o + (w8 ? w8_matrix_bytes(mk.M, mk.K) : w4_packed_bytes(mk.M, mk.K)) > arena_bytes)
          return set_error(MVB_ERR_ARG, "%s matrix %d of layer %d runs past the end of the arena", kind, t, l);
      }
    if (w8) {
      if (h->off[2] + w8_matrix_bytes(cfg->dim, cfg->spk_dim) > arena_bytes || h->off[4] + w8_matrix_bytes(cfg->vocab, cfg->dim) > arena_bytes)
        return set_error(MVB_ERR_ARG, "%s matrix speaker_cond_pos or lm_head runs past the end of the arena", kind);
      // lm_head's q, widened once: the head GEMM of every prefill chunk reads it from here; an fp8 engine's
      // speaker_cond_pos q too, for k_spk_proj
      h->w8_head = h->wsp<__nv_bfloat16>(h->L.w8_head);
      WidenBatch m{};
      m.src[0] = reinterpret_cast<const uint8_t*>(h->w(4));
      m.dst[0] = h->w8_head;
      m.M[0] = cfg->vocab; m.K[0] = cfg->dim; m.n = 1;
      if (fmt == WFmt::FP8) {
        h->f8_spk = h->wsp<__nv_bfloat16>(h->L.f8_spk);
        m.src[1] = reinterpret_cast<const uint8_t*>(h->w(2));
        m.dst[1] = h->f8_spk;
        m.M[1] = cfg->dim; m.K[1] = cfg->spk_dim; m.n = 2;
      }
      MVB_CK(widen(fmt, m, n_sm, 0));
      MVB_CK(cudaStreamSynchronize(0));
    }
  }
  S1State& s = h->st;
  s.slot_map = h->wsp<int>(h->L.slot_map);
  s.pos = h->wsp<int>(h->L.pos);
  s.row_tok = h->wsp<int>(h->L.row_tok);
  s.done = h->wsp<int>(h->L.done);
  s.n_gen = h->wsp<int>(h->L.n_gen);
  s.gen_tokens = h->wsp<int>(h->L.gen_tokens);
  s.sampled_tokens = h->wsp<int>(h->L.sampled);
  s.samp = h->wsp<SamplingDev>(h->L.samp);
  s.noise = h->wsp<const float*>(h->L.noise);
  s.forced = h->wsp<const int*>(h->L.forced);
  s.attn_ticket = h->wsp<unsigned>(h->L.ticket);
  s.budget = h->wsp<int>(h->L.budget);
  s.noise_base = h->wsp<int>(h->L.noise_base);
  s.max_new = cfg->max_new;
  s.block_size = cfg->block_size;
  h->path_b = !(cfg->options & MVB_S1_NO_ROWS_PATH);
  h->path_c = !(cfg->options & MVB_S1_NO_RESIDENT);
  h->fused = !(cfg->options & MVB_S1_UNFUSED_SAMPLER);
  h->trace = (cfg->options & MVB_S1_TRACE) != 0;
  {
    int* rb = h->wsp<int>(h->L.b_rows);
    h->rows.cache_row = rb; h->rows.pos = rb + RB_MAX; h->rows.tok = rb + 2 * RB_MAX; h->rows.utt = rb + 3 * RB_MAX;
    h->rows.cond = rb + 4 * RB_MAX;
    const int D = cfg->dim, F = cfg->intermediate;
    h->tmW.resize((size_t)cfg->n_layer * 5 + 1);
    bool ok = true;
    for (int l = 0; l < cfg->n_layer && ok; ++l) {
      ok = ok && make_tmap_bf16(&h->tmW[l * 5 + 0], h->tc_w(l, 1), 3 * D, D, 128);
      ok = ok && make_tmap_bf16(&h->tmW[l * 5 + 1], h->tc_w(l, 2), D, D, 128);
      ok = ok && make_tmap_bf16(&h->tmW[l * 5 + 2], h->tc_w(l, 4), F, D, 128);
      ok = ok && make_tmap_bf16(&h->tmW[l * 5 + 3], h->tc_w(l, h->gelu() ? 4 : 5), F, D, 128);   // GELU: c_fc again
      ok = ok && make_tmap_bf16(&h->tmW[l * 5 + 4], h->tc_w(l, 6), D, F, 128);
    }
    ok = ok && make_tmap_bf16(&h->tmW[(size_t)cfg->n_layer * 5], h->row_scaled() ? h->w8_head : h->w(4), cfg->vocab, D, 128);
    if (!ok) return set_error(MVB_ERR_CUDA, "cuTensorMapEncodeTiled failed for a weight matrix");
  }
  // The persistent kernel's bf16-cache attention fetches KV tiles through tm_kv as whole 64-position boxes: positions
  // past the valid ones must hold finite values, and the map must be encodable.  Where it is not, path C is declined.
  // It has no fp8-cache form: an fp8 cache never takes path C (kv_ok stays false).
  memset(&h->tm_kv, 0, sizeof(h->tm_kv));
  bool kv_ok = cfg->kv_dtype == MVB_KV_FP32;
  if (cfg->kv_dtype == MVB_KV_BF16 && cfg->block_size % 64 == 0) {
    MVB_CK(cudaMemset(h->kv, 0, (size_t)cfg->n_layer * 2 * h->kv_half_bytes()));
    const uint64_t rows = (uint64_t)cfg->n_layer * 2 * (h->kv_half_bytes() / 256);
    kv_ok = rows < (1ull << 31) && make_tmap_bf16(&h->tm_kv, h->kv, rows, 128, 64);
  }
  h->h_topk.assign(cfg->max_utts, 0);
  h->h_link.assign(cfg->max_utts, 0);
  h->voices.resize(1);
  h->voices[0].first_layer = cfg->n_layer + 1;
  h->next_voice.assign(cfg->max_utts, 0);
  h->slot_voice.assign(cfg->max_utts, 0);
  {
    // persistent decode kernel: needs a uniform layer stride (true for arenas packed in checkpoint order)
    const int D = cfg->dim, F = cfg->intermediate, V = cfg->vocab;
    // an int4, int8 or fp8 engine, and any architecture but the production one, never uses path C
    bool ok = cfg->n_layer >= 1 && fmt == WFmt::BF16 && kv_ok && h->production_arch() && default_staging_ok(*cfg);
    const int o0 = MVB_S1_GLOBAL_TENSORS;
    uint64_t stride = cfg->n_layer > 1 ? h->off[o0 + MVB_S1_LAYER_TENSORS] - h->off[o0] : 2 * (uint64_t)(4 * D * D + 3 * D * F + 2 * D);
    for (int l = 1; l < cfg->n_layer && ok; ++l)
      for (int t = 0; t < MVB_S1_LAYER_TENSORS; ++t)
        ok = ok && (h->off[o0 + l * MVB_S1_LAYER_TENSORS + t] - h->off[o0 + (l - 1) * MVB_S1_LAYER_TENSORS + t] == stride);
    ok = ok && (stride % 16 == 0);
    h->layer_stride_elems = stride / 2;
    const uint64_t NL = cfg->n_layer;
    const int rows = PcCfg<16>::TILE_ROWS;
    ok = ok && make_tmap_bf16_3d(&h->tm3[0], h->lw(0, 1), D, 3 * D, NL, stride, rows);
    ok = ok && make_tmap_bf16_3d(&h->tm3[1], h->lw(0, 2), D, D, NL, stride, rows);
    ok = ok && make_tmap_bf16_3d(&h->tm3[2], h->lw(0, 4), D, F, NL, stride, rows);
    ok = ok && make_tmap_bf16_3d(&h->tm3[3], h->lw(0, 5), D, F, NL, stride, rows);
    ok = ok && make_tmap_bf16_3d(&h->tm3[4], h->lw(0, 6), F, D, NL, stride, rows);
    ok = ok && make_tmap_bf16_3d(&h->tm3[5], h->w(4), D, V, 1, (uint64_t)V * D * 2, rows);
    h->pm[0] = plan_pc(3 * D, D, h->n_sm, rows);
    h->pm[1] = plan_pc(D, D, h->n_sm, rows);
    h->pm[2] = plan_pc(2 * F, D, h->n_sm, rows);
    h->pm[3] = plan_pc(D, F, h->n_sm, rows);
    h->pm[4] = plan_pc(V, D, h->n_sm, rows);
    for (int i = 0; i < 5; ++i) ok = ok && h->pm[i].S > 0;
    ok = ok && (F % rows == 0) && (D % rows == 0);     // w1 | w3 share one tile index space: F must be whole tiles
    h->pc_ok = ok;
  }
  // Opt-in shared-memory size is a per-device function attribute: set it for the device this handle lives on
  // (a process may hold engines on several GPUs).
#define MVB_PC_ATTR(FP, NBV)                                                                                        \
  MVB_CK(cudaFuncSetAttribute(k_decode_persistent<FP, NBV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PcCfg<NBV>::SMEM))
  MVB_PC_ATTR(true, 32); MVB_PC_ATTR(true, 16); MVB_PC_ATTR(false, 32); MVB_PC_ATTR(false, 16);
#undef MVB_PC_ATTR
  MVB_CK(cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking));
  MVB_CK(cudaMallocHost(&h->h_flags, sizeof(int) * 4 * 64));
  *out = hb.release();
  return MVB_OK;
}

extern "C" int mvb_s1_create_ex(const mvb_s1_config* cfg, const mvb_s1_arch* arch, const void* d_arena, size_t arena_bytes,
                                const uint64_t* offsets, void* d_kv, void* d_ws, mvb_s1** out) {
  return create_engine(cfg, arch, d_arena, arena_bytes, offsets, d_kv, d_ws, out, WFmt::BF16);
}

extern "C" int mvb_s1_create(const mvb_s1_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                             void* d_kv, void* d_ws, mvb_s1** out) {
  return mvb_s1_create_ex(cfg, nullptr, d_arena, arena_bytes, offsets, d_kv, d_ws, out);
}

extern "C" int mvb_s1_create_int4(const mvb_s1_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                                  void* d_kv, void* d_ws, mvb_s1** out) {
  return create_engine(cfg, nullptr, d_arena, arena_bytes, offsets, d_kv, d_ws, out, WFmt::INT4);
}

extern "C" int mvb_s1_create_int8(const mvb_s1_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                                  void* d_kv, void* d_ws, mvb_s1** out) {
  return create_engine(cfg, nullptr, d_arena, arena_bytes, offsets, d_kv, d_ws, out, WFmt::INT8);
}

extern "C" int mvb_s1_create_fp8(const mvb_s1_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                                 void* d_kv, void* d_ws, mvb_s1** out) {
  return create_engine(cfg, nullptr, d_arena, arena_bytes, offsets, d_kv, d_ws, out, WFmt::FP8);
}

extern "C" int mvb_s1_destroy(mvb_s1* h) {
  if (!h) return MVB_OK;
  for (auto& kv : h->graphs) cudaGraphExecDestroy(kv.second);
  for (auto& kv : h->vgraphs) cudaGraphExecDestroy(kv.second);
  for (auto& kv : h->vgraph_done) cudaEventDestroy(kv.second);
  if (h->vslots) cudaFree(h->vslots);
  if (h->vtickets) cudaFree(h->vtickets);
  if (h->d_tm) cudaFree(h->d_tm);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  if (h->h_flags) cudaFreeHost(h->h_flags);
  delete h;
  return MVB_OK;
}

extern "C" uint64_t mvb_s1_launch_count(const mvb_s1* h) { return h ? h->launches : 0; }

// ------------------------------------------------------------------------------------------------
static int gemv_grid(int n_items, int n_sm) {
  const int cap = 2 * n_sm * 8;                       // resident warps at 2 CTAs/SM
  const int ipw = (n_items + cap - 1) / cap;          // items per warp
  return (n_items + 8 * ipw - 1) / (8 * ipw);
}

// Launch with the programmatic-dependent-launch attribute: the kernel may start while its predecessor in the
// stream drains; it prefetches weights, then griddepcontrol.wait orders it after the predecessor's writes.
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// k_gemv_f8 over batch entries [0, n_utts): one launch row of up to F8_MAX_UTTS slots (gridDim.y > 1 only for a larger
// batch on an engine without the rows path), one n8 block of MMA columns up to 4 slots, two above.
template <int EPI>
static cudaError_t launch_gemv_f8(mvb_s1* h, cudaStream_t s, int n_utts, const GemvP& p, const S1State& st) {
  const dim3 grid(f8_gemv_ctas((p.M + 15) / 16, h->n_sm), (n_utts + F8_MAX_UTTS - 1) / F8_MAX_UTTS);
  h->launches++;
  if (n_utts > F8_MAX_UTTS / 2) return launch_pdl(k_gemv_f8<EPI, 2>, grid, dim3(256), 0, s, p, st, n_utts);
  return launch_pdl(k_gemv_f8<EPI, 1>, grid, dim3(256), 0, s, p, st, n_utts);
}

// p.W / p.W3 are matrices of format `fmt`: bf16 (k_gemv), int4 packed (k_gemv_w4), int8 (k_gemv_w8) or fp8 (k_gemv_f8);
// the first three take one item per warp and one utterance per launch row.  The LayerNorm prologue (`layer`, p.gain set),
// the Linear biases (p.bias set) and EPI_GELU exist for bf16 only.  A K whose staging rows need more than the default
// 48 KB of shared memory (a GELU c_proj, K = 4 dim) opts the bf16 instance in first.  `st` (default: the engine's
// decode state) supplies the slot map: batch entry i is slot st->slot_map[i].
template <int EPI>
static cudaError_t launch_gemv(mvb_s1* h, cudaStream_t s, int n_utts, const GemvP& p, WFmt fmt, bool layer,
                               const S1State* st = nullptr) {
  const S1State& state = st ? *st : h->st;
  const bool biased = p.bias != nullptr;
  const int n_items = (EPI == EPI_SWIGLU) ? p.M : p.M / 2;
  const dim3 grid(gemv_grid(n_items, h->n_sm), n_utts);
  const size_t smem = (size_t)2 * p.K * sizeof(float);
  if (fmt != WFmt::BF16) {
    if constexpr (EPI != EPI_GELU) {
      if (!layer && !biased) {
        if (fmt == WFmt::FP8) return launch_gemv_f8<EPI>(h, s, n_utts, p, state);
        h->launches++;
        return launch_pdl(fmt == WFmt::INT4 ? k_gemv_w4<EPI> : k_gemv_w8<EPI>, grid, dim3(256), smem, s, p, state);
      }
    }
    return cudaErrorInvalidValue;
  }
  void (*k)(GemvP, S1State) = layer ? (biased ? k_gemv<EPI, true, true> : k_gemv<EPI, true, false>)
                                    : (biased ? k_gemv<EPI, false, true> : k_gemv<EPI, false, false>);
  h->launches++;
  if (smem > 48 * 1024) {
    if (smem > GEMV_MAX_SMEM) return cudaErrorInvalidValue;
    const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  return launch_pdl(k, grid, dim3(256), smem, s, p, state);
}

// Attention of path A over layer l: the two CFG rows of n_utts utterances at their decode positions.  An fp8 cache first
// takes the new k / v from the projection's qkv rows (k_kv_store_f8); a bf16 / fp32 cache got them from its EPI_QKV
// scatter.
static int attn_decode(mvb_s1* h, cudaStream_t s, int n_utts, int l, const float* qkv, float* att) {
  const mvb_s1_config& c = h->cfg;
  const int D = c.dim, H = c.n_head;
  float* po = h->wsp<float>(h->L.part_o);
  float* pm = h->wsp<float>(h->L.part_ml);
  const dim3 ag(H, 2 * n_utts, ATT_SPLITS);
  if (h->kv_f8()) {
    const KvF8 kv = h->kv_f8_layer(l);
    MVB_CK(launch_pdl(k_kv_store_f8<false>, dim3((4 * n_utts * H + 7) / 8), dim3(256), 0, s, h->st, h->rows, 2 * n_utts, qkv,
                      kv, H, c.block_size, D));
    h->launches++;
    MVB_CK(launch_pdl(k_attn_decode_f8, ag, dim3(128), 0, s, h->st, qkv, kv, po, pm, att, H, c.block_size, D));
  } else {
    const char* kc = h->kv + (size_t)l * 2 * h->kv_half_bytes();
    const void* vc = kc + h->kv_half_bytes();
    if (c.kv_dtype == MVB_KV_FP32)
      MVB_CK(launch_pdl(k_attn_decode<true>, ag, dim3(128), 0, s, h->st, qkv, (const void*)kc, vc, po, pm, att, H, c.block_size, D));
    else
      MVB_CK(launch_pdl(k_attn_decode<false>, ag, dim3(128), 0, s, h->st, qkv, (const void*)kc, vc, po, pm, att, H, c.block_size, D));
  }
  h->launches++;
  return MVB_OK;
}

// The weight sets of one layer (l == n_layer: ln_f and the head) over a voice-grouped batch: the leading groups still on
// the base weights merge into one unit, every later group is a unit of its own.  Without a plan (every entry on voice
// 0): one unit, the whole batch on the base weights.
struct VUnit { int lo, hi, voice; };   // entries [lo, hi) of the grouped order
static int voice_units(const mvb_s1* h, const VoicePlan* vp, int n, int l, VUnit* u) {
  if (!vp) { u[0] = VUnit{0, n, 0}; return 1; }
  int g = 0, k = 0;
  while (g < vp->n && h->first_layer(vp->voice[g]) > l) ++g;
  if (g > 0) u[k++] = VUnit{0, vp->start[g], 0};
  for (; g < vp->n; ++g) u[k++] = VUnit{vp->start[g], vp->start[g + 1], vp->voice[g]};
  return k;
}

// Path A's decode state for a unit: a slice of the grouped slot map, or the engine's own state for the whole batch.
static S1State unit_state(const mvb_s1* h, const VUnit& u, int n) {
  S1State st = h->st;
  if (u.lo != 0 || u.hi != n) st.slot_map = h->vslots + u.lo;
  return st;
}

// One forward position for `n_utts` logical utterances (layers/combined.py:38-50 per layer, model.py:303 ln_f, the tied
// head model.py:137-143): embed, then per layer ln_1 -> c_attn (+ bias) + cache scatter, attention, c_proj (+ bias) +
// residual, ln_2 -> SwiGLU or GELU MLP (+ biases), mlp.c_proj (+ bias) + residual; then ln_f -> head.  The norms are
// RMSNorm or LayerNorm (eps 1e-5, beta); the production architecture is RMSNorm, SwiGLU and no bias.  With a voice
// plan every projection runs once per unit (voice_units) over that unit's slots; the attention runs once for all.
static int launch_body(mvb_s1* h, cudaStream_t s, int n_utts, const VoicePlan* vp = nullptr) {
  const mvb_s1_config& c = h->cfg;
  const int D = c.dim, F = c.intermediate, V = c.vocab, H = c.n_head;
  const bool ln = h->layer_norm();
  const float eps = h->norm_eps();
  float* x = h->wsp<float>(h->L.x);
  float* qkv = h->wsp<float>(h->L.qkv);
  float* att = h->wsp<float>(h->L.att);
  float* ffn = h->wsp<float>(h->L.ffn);
  float* logits = h->wsp<float>(h->L.logits);
  MVB_CK(launch_pdl(k_embed, dim3(2, n_utts), dim3(256), 0, s, h->st, h->w(0), h->w(1),
                (const float*)h->wsp<float>(h->L.spk), x, D));
  h->launches++;
  const size_t half = h->kv_half_bytes();
  VUnit us[MVB_S1_MAX_VOICES];
  for (int l = 0; l < c.n_layer; ++l) {
    char* kc = h->kv + (size_t)l * 2 * half;
    char* vc = kc + half;
    const int nu = voice_units(h, vp, n_utts, l, us);
    // ln_1 + c_attn + cache scatter (fp8 cache: the qkv rows only)
    for (int i = 0; i < nu; ++i) {
      const int v = us[i].voice, n = us[i].hi - us[i].lo;
      const S1LayerP& lp = h->vlp(v, l);
      const S1State st = unit_state(h, us[i], n_utts);
      GemvP p{};
      p.eps = eps;
      p.W = h->vlw(v, l, 1); p.x = x; p.ldx = D; p.gain = lp.g1; p.beta = lp.b1; p.bias = lp.qkv_b;
      p.out = qkv; p.ldo = 3 * D; p.M = 3 * D; p.K = D;
      p.kcache = kc; p.vcache = vc; p.H = H; p.S_max = c.block_size; p.D = D; p.kv_fp32 = c.kv_dtype == MVB_KV_FP32;
      MVB_CK(h->kv_f8() ? launch_gemv<EPI_STORE>(h, s, n, p, h->fmt, ln, &st) : launch_gemv<EPI_QKV>(h, s, n, p, h->fmt, ln, &st));
    }
    // attention over [0, pos]
    if (int e = attn_decode(h, s, n_utts, l, qkv, att)) return e;
    for (int i = 0; i < nu; ++i) {
      const int v = us[i].voice, n = us[i].hi - us[i].lo;
      const S1LayerP& lp = h->vlp(v, l);
      const S1State st = unit_state(h, us[i], n_utts);
      // c_proj + residual
      GemvP p{};
      p.eps = eps;
      p.W = h->vlw(v, l, 2); p.x = att; p.ldx = D; p.bias = lp.o_b; p.out = x; p.ldo = D; p.M = D; p.K = D;
      MVB_CK(launch_gemv<EPI_RESID>(h, s, n, p, h->fmt, false, &st));
      // ln_2 + GELU(c_fc x) or silu(w1 x) * w3 x
      p = GemvP{};
      p.eps = eps;
      p.W = h->vlw(v, l, 4); p.x = x; p.ldx = D; p.gain = lp.g2; p.beta = lp.b2; p.bias = lp.fc_b; p.out = ffn; p.ldo = F;
      p.M = F; p.K = D;
      if (h->gelu()) {
        MVB_CK(launch_gemv<EPI_GELU>(h, s, n, p, h->fmt, ln, &st));
      } else {
        p.W3 = h->vlw(v, l, 5); p.bias3 = lp.fc3_b;
        MVB_CK(launch_gemv<EPI_SWIGLU>(h, s, n, p, h->fmt, ln, &st));
      }
      // mlp.c_proj + residual
      p = GemvP{};
      p.eps = eps;
      p.W = h->vlw(v, l, 6); p.x = ffn; p.ldx = F; p.bias = lp.proj_b; p.out = x; p.ldo = D; p.M = D; p.K = F;
      MVB_CK(launch_gemv<EPI_RESID>(h, s, n, p, h->fmt, false, &st));
    }
  }
  const int nu = voice_units(h, vp, n_utts, c.n_layer, us);
  for (int i = 0; i < nu; ++i) {
    const int v = us[i].voice;
    const S1State st = unit_state(h, us[i], n_utts);
    GemvP p{};
    p.eps = eps;
    p.W = h->w(4); p.x = x; p.ldx = D; p.gain = h->lnf_gain(v); p.beta = h->lnf_beta(v); p.out = logits; p.ldo = V; p.M = V;
    p.K = D;
    MVB_CK(launch_gemv<EPI_STORE>(h, s, us[i].hi - us[i].lo, p, h->head_fmt(), ln, &st));
  }
  return MVB_OK;
}


// ------------------------------------------------------------------------------------------------
// Path B: the same forward pass for R arbitrary activation rows on the tensor cores (tc_gemm, linear.cu).
// Used for batched decode (R = 2 * n_utts) and for prefill chunks (R = 2 * tokens).
static const CUtensorMap* tmap_b(mvb_s1* h, int NB, int K) {
  auto key = std::make_pair(NB, K);
  auto it = h->tmB.find(key);
  if (it == h->tmB.end()) {
    CUtensorMap tm;
    if (!make_tmap_bf16(&tm, h->wsp<char>(h->L.b_B), (uint64_t)NB, (uint64_t)K, (uint32_t)NB)) return nullptr;
    it = h->tmB.emplace(key, tm).first;
  }
  return &it->second;
}

struct LinB {
  const float* x; int ldx; const __nv_bfloat16* gain;  // input rows (+ optional norm gain: the architecture's norm)
  const CUtensorMap* tmW; const CUtensorMap* tmW3;     // tensor maps of W (and W3 for SwiGLU)
  int M, K;
  float* out; int ldo;
  const __nv_bfloat16* scale = nullptr;                // int8 / fp8 engine: row scales of W (and W3)
  const __nv_bfloat16* scale3 = nullptr;
  const __nv_bfloat16* beta = nullptr;                 // LayerNorm with bias: the norm's beta
  const __nv_bfloat16* bias = nullptr;                 // Linear biases of W (and W3)
  const __nv_bfloat16* bias3 = nullptr;
};

template <int EPI>
static int linear_b(mvb_s1* h, cudaStream_t s, int R, const LinB& a, void* kc = nullptr, void* vc = nullptr) {
  const mvb_s1_config& c = h->cfg;
  TcGemm g{};
  g.epi = EPI; g.R = R; g.Rpad = (R + 15) / 16 * 16; g.split_lo = 1;   // activations as hi + lo bf16 terms
  g.tmB = tmap_b(h, 2 * g.Rpad, a.K);
  if (!g.tmB) return set_error(MVB_ERR_CUDA, "cuTensorMapEncodeTiled failed for the activation buffer");
  g.tmW = a.tmW; g.tmW3 = a.tmW3;
  g.B = h->wsp<__nv_bfloat16>(h->L.b_B);
  g.x = a.x; g.ldx = a.ldx; g.gain = a.gain; g.eps = c.norm_eps;
  if (a.gain != nullptr && h->layer_norm()) {   // LayerNorm (layers/layers.py:8-17): eps 1e-5, optional beta
    g.layer_norm = 1; g.beta = a.beta; g.eps = 1e-5f;
  }
  g.M = a.M; g.K = a.K; g.out = a.out; g.ldo = a.ldo;
  g.kcache = kc; g.vcache = vc; g.row_cache = h->rows.cache_row; g.row_pos = h->rows.pos;
  g.H = c.n_head; g.S_max = c.block_size; g.D = c.dim; g.kv_fp32 = c.kv_dtype == MVB_KV_FP32;
  g.scratch = h->wsp<float>(h->L.b_scratch);
  g.tickets = h->wsp<unsigned>(h->L.b_tickets);
  g.n_sm = h->n_sm;
  g.scale = a.scale; g.scale3 = a.scale3;
  g.bias = a.bias; g.bias3 = a.bias3;
  MVB_CK(tc_gemm(s, g));
  h->launches += 2;   // k_prep_b + k_tc_gemm
  return MVB_OK;
}

// One projection of a voice-grouped decode batch (rows in batch order, h->row_grp filled by k_voice_rows): unit i of
// `us` multiplies its rows by its weights (a[i]: tensor maps, norm gain / beta, biases; `dtm[i]` / `dtm3[i]`: the same
// maps in device memory) in one grouped launch.  One unit is the ungrouped linear_b over every row.
template <int EPI>
static int linear_units(mvb_s1* h, cudaStream_t s, int R, const VoicePlan* vp, const VUnit* us, int nu, const LinB* a,
                        const CUtensorMap* const* dtm, const CUtensorMap* const* dtm3, void* kc = nullptr, void* vc = nullptr) {
  if (nu == 1) return linear_b<EPI>(h, s, R, a[0], kc, vc);
  const mvb_s1_config& c = h->cfg;
  TcGemm g{};
  g.epi = EPI; g.R = R; g.Rpad = (R + 15) / 16 * 16; g.split_lo = 1;
  g.tmB = tmap_b(h, 2 * g.Rpad, a[0].K);
  if (!g.tmB) return set_error(MVB_ERR_CUDA, "cuTensorMapEncodeTiled failed for the activation buffer");
  g.B = h->wsp<__nv_bfloat16>(h->L.b_B);
  g.x = a[0].x; g.ldx = a[0].ldx; g.eps = c.norm_eps;
  if (a[0].gain != nullptr && h->layer_norm()) { g.layer_norm = 1; g.eps = 1e-5f; }
  g.M = a[0].M; g.K = a[0].K; g.out = a[0].out; g.ldo = a[0].ldo;
  g.kcache = kc; g.vcache = vc; g.row_cache = h->rows.cache_row; g.row_pos = h->rows.pos;
  g.H = c.n_head; g.S_max = c.block_size; g.D = c.dim; g.kv_fp32 = c.kv_dtype == MVB_KV_FP32;
  g.scratch = h->wsp<float>(h->L.b_scratch);
  g.n_sm = h->n_sm;
  TcGemmGrp q{};
  q.row_grp = h->row_grp;
  q.tickets = h->vtickets;
  q.n_units = nu;
  for (int gi = 0; gi < vp->n; ++gi)
    for (int i = 0; i < nu; ++i)
      if (vp->start[gi] >= us[i].lo && vp->start[gi] < us[i].hi) q.g2u[gi] = q.prep_g2u[gi] = i;
  for (int i = 0; i < nu; ++i) {
    q.tmW[i] = dtm[i]; q.tmW3[i] = dtm3[i]; q.bias[i] = a[i].bias; q.bias3[i] = a[i].bias3;
    q.gain[i] = a[i].gain; q.beta[i] = a[i].beta;
  }
  MVB_CK(tc_gemm_grouped(s, g, q));
  h->launches += 2;   // k_prep_b_grp + k_tc_gemm_grp
  return MVB_OK;
}

// The qkv projection of path B (operands a[i] of each unit) and the attention of the R rows of h->rows over layer l's
// cache.  An fp8 cache takes the new k / v from the stored qkv rows (G_STORE, then k_kv_store_f8) before the attention
// reads them: a prefill chunk attends to its own positions.
static int qkv_attn_rows(mvb_s1* h, cudaStream_t s, int R, int l, const VoicePlan* vp, const VUnit* us, int nu, const LinB* a,
                         const CUtensorMap* const* dtm, const float* qkv, float* att) {
  const mvb_s1_config& c = h->cfg;
  const int D = c.dim, H = c.n_head;
  char* kc = h->kv + (size_t)l * 2 * h->kv_half_bytes();
  char* vc = kc + h->kv_half_bytes();
  float* po = h->wsp<float>(h->L.b_part_o);
  float* pm = h->wsp<float>(h->L.b_part_ml);
  unsigned* tk = h->wsp<unsigned>(h->L.b_att_tickets);
  dim3 ag(H, R, ATT_SPLITS);
  if (h->kv_f8()) {
    if (int e = linear_units<G_STORE>(h, s, R, vp, us, nu, a, dtm, dtm)) return e;
    const KvF8 kv = h->kv_f8_layer(l);
    k_kv_store_f8<true><<<(2 * R * H + 7) / 8, 256, 0, s>>>(h->st, h->rows, R, qkv, kv, H, c.block_size, D);
    h->launches++;
    MVB_CK(cudaGetLastError());
    k_attn_rows_f8<<<ag, 128, 0, s>>>(h->rows, qkv, kv, po, pm, tk, att, H, c.block_size, D);
  } else {
    if (int e = linear_units<G_QKV>(h, s, R, vp, us, nu, a, dtm, dtm, kc, vc)) return e;
    if (c.kv_dtype == MVB_KV_FP32)
      k_attn_rows<true><<<ag, 128, 0, s>>>(h->rows, qkv, kc, vc, po, pm, tk, att, H, c.block_size, D);
    else
      k_attn_rows<false><<<ag, 128, 0, s>>>(h->rows, qkv, kc, vc, po, pm, tk, att, H, c.block_size, D);
  }
  h->launches++;
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

// The final norm and the head of path B over R rows of x: y = ln_f(x) . lm_head^T into out [R, vocab].  A prefill runs on
// one voice (`voice`); a voice-grouped decode batch (vp) normalises each row with its voice's ln_f and then runs ONE
// GEMM over every row, since lm_head is shared by every voice.
static int head_b(mvb_s1* h, cudaStream_t s, int R, const float* x, float* out, int voice = 0, const VoicePlan* vp = nullptr) {
  const mvb_s1_config& c = h->cfg;
  if (!vp) {
    const CUtensorMap* tm = h->vtm(voice, c.n_layer, 0);
    LinB a{x, c.dim, h->lnf_gain(voice), tm, tm, c.vocab, c.dim, out, c.vocab, h->head_scale()};
    a.beta = h->lnf_beta(voice);
    return linear_b<G_STORE>(h, s, R, a);
  }
  TcGemm g{};
  g.epi = G_STORE; g.R = R; g.Rpad = (R + 15) / 16 * 16; g.split_lo = 1;
  g.tmB = tmap_b(h, 2 * g.Rpad, c.dim);
  if (!g.tmB) return set_error(MVB_ERR_CUDA, "cuTensorMapEncodeTiled failed for the activation buffer");
  g.B = h->wsp<__nv_bfloat16>(h->L.b_B);
  g.x = x; g.ldx = c.dim; g.eps = c.norm_eps;
  if (h->layer_norm()) { g.layer_norm = 1; g.eps = 1e-5f; }
  g.M = c.vocab; g.K = c.dim; g.out = out; g.ldo = c.vocab;
  g.scratch = h->wsp<float>(h->L.b_scratch);
  g.n_sm = h->n_sm;
  TcGemmGrp q{};
  q.row_grp = h->row_grp;
  q.tickets = h->vtickets;
  q.n_units = 1;
  q.tmW[0] = q.tmW3[0] = h->voice_tm(0, c.n_layer, 0);
  for (int gi = 0; gi < vp->n; ++gi) {
    q.prep_g2u[gi] = gi;
    q.gain[gi] = h->lnf_gain(vp->voice[gi]);
    q.beta[gi] = h->lnf_beta(vp->voice[gi]);
  }
  MVB_CK(tc_gemm_grouped(s, g, q));
  h->launches += 2;
  return MVB_OK;
}

// embed + all layers for the R rows described by h->rows (already filled on the device): path A's projections with the
// LayerNorm prologue of k_prep_b<true> and the BIASED / G_GELU / SCALED epilogues of k_tc_gemm.  A prefill runs on one
// voice (`voice`).  A voice-grouped decode batch (vp, rows in batch order, row_grp filled) runs each projection as one
// grouped launch over its units (voice_units): one unit, i.e. every layer below the lowest first_layer in the batch, is
// the ungrouped launch.
static int launch_layers_b(mvb_s1* h, cudaStream_t s, int R, int voice = 0, const VoicePlan* vp = nullptr) {
  const mvb_s1_config& c = h->cfg;
  const int D = c.dim, F = c.intermediate;
  float* x = h->wsp<float>(h->L.b_x);
  float* qkv = h->wsp<float>(h->L.b_qkv);
  float* att = h->wsp<float>(h->L.b_att);
  float* ffn = h->wsp<float>(h->L.b_ffn);
  k_embed_rows<<<R, 256, 0, s>>>(h->rows, h->w(0), h->w(1), h->wsp<float>(h->L.spk), x, D);
  h->launches++;
  MVB_CK(cudaGetLastError());
  VUnit us[MVB_S1_MAX_VOICES];
  LinB qa[MVB_S1_MAX_VOICES], oa[MVB_S1_MAX_VOICES], fa[MVB_S1_MAX_VOICES], pa[MVB_S1_MAX_VOICES];
  const CUtensorMap* dt[5][MVB_S1_MAX_VOICES];
  for (int l = 0; l < c.n_layer; ++l) {
    if (h->fmt != WFmt::BF16) {   // this layer's W_deq (int4) or q (int8, fp8) -> the scratch the tensor maps of every layer point at
      WidenBatch m{};
      const int ts[5] = {1, 2, 4, 5, 6};
      for (int i = 0; i < 5; ++i) {
        const Mk mk = layer_mk(c, ts[i]);
        m.src[i] = reinterpret_cast<const uint8_t*>(h->lw(l, ts[i]));
        m.dst[i] = const_cast<__nv_bfloat16*>(h->tc_w(l, ts[i]));
        m.M[i] = mk.M; m.K[i] = mk.K;
      }
      m.n = 5;
      h->launches++;
      MVB_CK(widen(h->fmt, m, h->n_sm, s));
    }
    int nu = 1;
    if (vp) nu = voice_units(h, vp, R / 2, l, us);
    else us[0] = VUnit{0, R / 2, voice};
    for (int i = 0; i < nu; ++i) {
      const int v = us[i].voice;
      const S1LayerP& p = h->vlp(v, l);
      qa[i] = LinB{x, D, p.g1, h->vtm(v, l, 0), h->vtm(v, l, 0), 3 * D, D, qkv, 3 * D, h->tc_lscale(l, 1)};
      qa[i].beta = p.b1; qa[i].bias = p.qkv_b;
      oa[i] = LinB{att, D, nullptr, h->vtm(v, l, 1), h->vtm(v, l, 1), D, D, x, D, h->tc_lscale(l, 2)};
      oa[i].bias = p.o_b;
      fa[i] = LinB{x, D, p.g2, h->vtm(v, l, 2), h->vtm(v, l, 3), F, D, ffn, F, h->tc_lscale(l, 4), h->tc_lscale(l, 5)};
      fa[i].beta = p.b2; fa[i].bias = p.fc_b; fa[i].bias3 = p.fc3_b;
      pa[i] = LinB{ffn, F, nullptr, h->vtm(v, l, 4), h->vtm(v, l, 4), D, F, x, D, h->tc_lscale(l, 6)};
      pa[i].bias = p.proj_b;
      for (int t = 0; t < 5; ++t) dt[t][i] = nu > 1 ? h->voice_tm(v, l, t) : nullptr;
    }
    if (int e = qkv_attn_rows(h, s, R, l, vp, us, nu, qa, dt[0], qkv, att)) return e;
    if (int e = linear_units<G_RESID>(h, s, R, vp, us, nu, oa, dt[1], dt[1])) return e;
    if (int e = h->gelu() ? linear_units<G_GELU>(h, s, R, vp, us, nu, fa, dt[2], dt[2])
                          : linear_units<G_SWIGLU>(h, s, R, vp, us, nu, fa, dt[2], dt[3]))
      return e;
    if (int e = linear_units<G_RESID>(h, s, R, vp, us, nu, pa, dt[4], dt[4])) return e;
  }
  return MVB_OK;
}

// batched decode position: rows from the decode state (batch order), logits land in the sampler's buffer.  With a voice
// plan, k_voice_rows first records each row's voice group for the grouped launches.
static int launch_body_b(mvb_s1* h, cudaStream_t s, int n_utts, const VoicePlan* vp = nullptr) {
  const int R = 2 * n_utts;
  k_rows_decode<<<1, 128, 0, s>>>(h->st, h->rows, n_utts);
  h->launches++;
  MVB_CK(cudaGetLastError());
  if (vp) {
    VoiceRows vr{};
    for (int i = 0; i < n_utts; ++i) vr.grp[i] = vp->grp[i];
    k_voice_rows<<<1, 128, 0, s>>>(vr, R, h->row_grp);
    h->launches++;
    MVB_CK(cudaGetLastError());
  }
  if (int e = launch_layers_b(h, s, R, 0, vp)) return e;
  return head_b(h, s, R, h->wsp<float>(h->L.b_x), h->wsp<float>(h->L.logits), 0, vp);
}


// ------------------------------------------------------------------------------------------------
// Path C: one persistent kernel per decode position (decode_persistent.cuh) followed by the sampler.
static int launch_persistent(mvb_s1* h, cudaStream_t s, int n_utts, int n_steps, bool fused) {
  const mvb_s1_config& c = h->cfg;
  PcParams p{};
  p.n_layer = c.n_layer; p.D = c.dim; p.F = c.intermediate; p.V = c.vocab; p.H = c.n_head; p.S_max = c.block_size;
  p.n_steps = n_steps; p.fused = fused ? 1 : 0;
  p.R = 2 * n_utts; p.n_utts = n_utts; p.kv_fp32 = c.kv_dtype == MVB_KV_FP32; p.eps = c.norm_eps;
  p.m_qkv = h->pm[0]; p.m_o = h->pm[1]; p.m_w13 = h->pm[2]; p.m_w2 = h->pm[3]; p.m_head = h->pm[4];
  p.attn_norm = h->lw(0, 0); p.ffn_norm = h->lw(0, 3); p.out_norm = h->w(3);
  p.layer_stride = h->layer_stride_elems;
  p.tok_emb = h->w(0); p.pos_emb = h->w(1); p.spk_proj = h->wsp<float>(h->L.spk);
  p.x = h->wsp<float>(h->L.c_x); p.qkv = h->wsp<float>(h->L.c_qkv); p.gu = h->wsp<float>(h->L.c_gu);
  p.logits = h->wsp<float>(h->L.logits);
  p.part_o = h->wsp<float>(h->L.c_part_o); p.part_ml = h->wsp<float>(h->L.c_part_ml);
  p.stat = h->wsp<float>(h->L.c_stat);
  p.samp_part = h->wsp<float>(h->L.c_samp_part);
  p.samp_best = h->wsp<unsigned long long>(h->L.c_samp_best);
  p.kv = h->kv; p.kv_half = h->kv_half_bytes();
  p.kv_rows_half = (long long)(h->kv_half_bytes() / 256);
  p.bar = h->wsp<unsigned>(h->L.c_bar);
  p.trace = (h->trace && h->n_sm <= 160) ? h->wsp<long long>(h->L.c_trace) : nullptr;
  p.st = h->st;
  // launch-time invariants of the kernel: grid-barrier counter, RMSNorm statistics and arg-max slots start from zero
  MVB_CK(cudaMemsetAsync(p.bar, 0, 4, s));
  MVB_CK(cudaMemsetAsync(p.stat, 0, sizeof(float) * (size_t)(2 * c.n_layer + 1) * PC_RPAD, s));
  MVB_CK(cudaMemsetAsync(p.samp_best, 0, sizeof(unsigned long long) * 2 * (PC_RPAD / 2), s));
  h->launches++;
  const bool fp = p.kv_fp32 != 0, wide = p.R > 8;
  const CUtensorMap* tm = h->tm3;
#define MVB_PC_LAUNCH(FP, NBV)                                                                                        \
  MVB_CK(launch_pdl(k_decode_persistent<FP, NBV>, dim3(h->n_sm), dim3(PC_THREADS), PcCfg<NBV>::SMEM, s,                   \
                tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], h->tm_kv, p))
  if (fp && wide) MVB_PC_LAUNCH(true, 32);
  else if (fp) MVB_PC_LAUNCH(true, 16);
  else if (wide) MVB_PC_LAUNCH(false, 32);
  else MVB_PC_LAUNCH(false, 16);
#undef MVB_PC_LAUNCH
  return MVB_OK;
}

// Host-side capacity check of the persistent kernel's per-CTA attention tile table (build_att_table, which traps once a
// CTA would own more than PC_MAX_TILES tiles).  With G = n_sm CTAs, R = 2 n_utts rows, ppc positions per tile and
// zmax = max(1, G / (R H)), a row of L <= block_size positions has tt = ceil(L / ppc) <= TT = ceil(block_size / ppc)
// tiles, cut into nz = ceil(tt / tps) splits of tps = ceil(tt / min(zmax, tt)) tiles.  Then
//   nz <= min(zmax, tt) <= Z = min(zmax, TT)        (tps >= tt / min(zmax, tt)), and
//   tps <= ceil(TT / Z)                             (tps = 1 while tt <= zmax, else ceil(tt / zmax) <= ceil(TT / zmax)),
// so the batch has at most R H Z units of at most ceil(TT / Z) tiles each.  Units are dealt round-robin over the G CTAs,
// so no CTA owns more than ceil(R H Z / G) units, i.e. ceil(R H Z / G) * ceil(TT / Z) tiles, whatever the positions.
// The same Z bounds the split count that indexes the PC_MAX_CHUNKS partial slots of every (row, head).
// The bound is derived for G = n_sm, so which batches reach PC_MAX_TILES depends on the part.  At block_size 2048, H = 16
// it is reached (exactly 128 tiles) by fp32 KV with 8 utterances at 132 SMs, fp32 with 1 utterance at 16, fp32 with 4 at
// 64, bf16 with 8 at 64 and bf16 with 1 at 8; a batch one past such an edge goes to the per-layer path.
static bool pc_att_fits(const mvb_s1* h, int n_utts) {
  const int R = 2 * n_utts, H = h->cfg.n_head, G = h->n_sm;
  const int ppc = PC_KV_TILE_BYTES / (128 * (int)h->kv_elem());
  const long long TT = (h->cfg.block_size + ppc - 1) / ppc;
  const long long zmax = G / (R * H) > 1 ? G / (R * H) : 1;
  const long long Z = zmax < TT ? zmax : TT;
  const long long units_per_cta = ((long long)R * H * Z + G - 1) / G;
  return Z <= PC_MAX_CHUNKS && units_per_cta * ((TT + Z - 1) / Z) <= PC_MAX_TILES;
}

// Slots [0, n_utts) are all on voice 0: the only batches the resident decode kernel serves (it walks the base arena
// with one uniform layer stride).
static bool all_base_voice(const mvb_s1* h, int n_utts) {
  for (int u = 0; u < n_utts; ++u)
    if (h->slot_voice[u] != 0) return false;
  return true;
}

// The persistent decode kernel serves the batch (else the per-layer path does).  CTA 2b alone writes batch entry b's
// x rows and decode state back (decode_persistent.cuh, `owner`), so CTA 2 (n_utts - 1) must exist: pc_att_fits does not
// imply it at a short block_size or a small width.
static bool use_path_c(const mvb_s1* h, int n_utts) {
  return h->path_c && h->pc_ok && 2 * n_utts <= PC_RPAD && 2 * n_utts - 1 <= h->n_sm && pc_att_fits(h, n_utts) &&
         all_base_voice(h, n_utts);
}

// The voice plan of a batch: entry i is slot `utt` (a single-entry prefill position) or slot i (decode).  False, and no
// plan, when every entry is on voice 0.  *order receives the entries in group order, *key the graph key.
static bool voice_plan(const mvb_s1* h, int n_utts, int utt, bool use_b, VoicePlan* vp, VoiceOrder* order,
                       std::vector<int>* key) {
  std::vector<int> ev(n_utts);
  bool any = false;
  for (int i = 0; i < n_utts; ++i) {
    ev[i] = h->slot_voice[utt >= 0 ? utt : i];
    any = any || ev[i] != 0;
  }
  if (!any) return false;
  std::vector<int> vs(ev.begin(), ev.end());
  std::sort(vs.begin(), vs.end());
  vs.erase(std::unique(vs.begin(), vs.end()), vs.end());
  std::stable_sort(vs.begin(), vs.end(), [&](int a, int b) { return h->first_layer(a) > h->first_layer(b); });
  vp->n = (int)vs.size();
  order->n = 0;
  for (int g = 0; g < vp->n; ++g) {
    vp->voice[g] = vs[g];
    vp->start[g] = order->n;
    for (int i = 0; i < n_utts; ++i)
      if (ev[i] == vs[g]) {
        order->entry[order->n++] = i;
        vp->grp[i] = g;
      }
  }
  vp->start[vp->n] = order->n;
  key->assign({use_b ? 1 : 0, n_utts});
  key->insert(key->end(), ev.begin(), ev.end());
  return true;
}

// One decode position of n_utts entries through a cached CUDA graph.  Batches whose entries are all on voice 0 are
// keyed by size and path, as they always were.  Any other batch is keyed by its voice of every entry too, since the
// grouping is part of the captured launches (path A's slot order and unit sizes, path B's row groups, every unit's
// weights): at most
// VOICE_GRAPHS_MAX such graphs are kept, the oldest destroyed first, so a batcher churning through voices holds at most
// 2 max_utts base graphs + VOICE_GRAPHS_MAX voice graphs, and re-captures (one capture per new grouping) beyond that.
static int run_body(mvb_s1* h, cudaStream_t s, int n_utts, bool allow_b = true, int utt = -1) {
  // Path A (CUDA-core GEMV) streams the weights once per utterance; from 2 utterances up the tensor-core
  // rows path streams them once per step for the whole batch.  slot_map must be the identity for path B
  // (its logits rows are batch-ordered), which mvb_s1_decode guarantees.  int4 / int8 decode: always path A.  fp8
  // decode: path A, whose k_gemv_f8 reads the weights once per step for up to F8_MAX_UTTS slots; a larger batch takes
  // path B, since one k_gemv_f8 launch row holds at most F8_MAX_UTTS slots (two n8 MMA blocks).
  const bool use_b = allow_b && h->path_b &&
                     ((h->fmt == WFmt::BF16 && n_utts >= 2) || (h->fmt == WFmt::FP8 && n_utts > F8_MAX_UTTS));
  VoicePlan vp;
  VoiceOrder order;
  std::vector<int> vkey;
  if (voice_plan(h, n_utts, utt, use_b, &vp, &order, &vkey)) {
    auto body = [&](cudaStream_t st) -> int {
      if (!use_b) {   // path A's units are slices of the grouped slot map; path B keeps the batch order
        k_voice_slots<<<1, 64, 0, st>>>(h->st.slot_map, order, h->vslots);
        h->launches++;
        MVB_CK(cudaGetLastError());
      }
      return use_b ? launch_body_b(h, st, n_utts, &vp) : launch_body(h, st, n_utts, &vp);
    };
    auto it = h->vgraphs.find(vkey);
    if (it == h->vgraphs.end()) {
      if ((int)h->vgraphs.size() >= VOICE_GRAPHS_MAX) {
        // the oldest graph's last launch (on whichever stream) must have finished before it is freed
        const std::vector<int> old = h->vgraph_age.front();
        h->vgraph_age.pop_front();
        MVB_CK(cudaEventSynchronize(h->vgraph_done[old]));
        cudaEventDestroy(h->vgraph_done[old]);
        cudaGraphExecDestroy(h->vgraphs[old]);
        h->vgraphs.erase(old);
        h->vgraph_nodes.erase(old);
        h->vgraph_done.erase(old);
      }
      const uint64_t before = h->launches;
      cudaGraphExec_t ge;
      const int e = capture_graph(h->cap_stream, &ge, body);
      h->vgraph_nodes[vkey] = (int)(h->launches - before);
      h->launches = before;
      if (e) return e;
      cudaEvent_t ev;
      if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) {
        cudaGraphExecDestroy(ge);
        return set_error(MVB_ERR_CUDA, "cudaEventCreate failed");
      }
      it = h->vgraphs.emplace(vkey, ge).first;
      h->vgraph_done[vkey] = ev;
      h->vgraph_age.push_back(vkey);
    }
    MVB_CK(cudaGraphLaunch(it->second, s));
    MVB_CK(cudaEventRecord(h->vgraph_done[vkey], s));
    h->launches += h->vgraph_nodes[vkey];
    return MVB_OK;
  }
  auto body = [&](cudaStream_t st) { return use_b ? launch_body_b(h, st, n_utts) : launch_body(h, st, n_utts); };
  const int key = n_utts + (use_b ? 1000 : 0);
  auto it = h->graphs.find(key);
  if (it == h->graphs.end()) {
    const uint64_t before = h->launches;
    cudaGraphExec_t ge;
    const int e = capture_graph(h->cap_stream, &ge, body);
    h->graph_nodes[key] = (int)(h->launches - before);
    h->launches = before;
    if (e) return e;
    it = h->graphs.emplace(key, ge).first;
  }
  MVB_CK(cudaGraphLaunch(it->second, s));
  h->launches += h->graph_nodes[key];
  return MVB_OK;
}

static SamplingDev to_dev(const mvb_sampling* p) {
  SamplingDev d;
  d.guidance = p->guidance_scale;
  d.temperature = p->temperature;
  d.top_p = p->top_p;
  d.top_k = p->top_k;
  d.end_of_audio = p->end_of_audio;
  d.link = 0;
  d.seed = p->seed;
  return d;
}

static int check_slot(const mvb_s1* h, int32_t utt) {   // every caller-supplied utterance slot must be one of the handle's
  return utt < 0 || utt >= h->cfg.max_utts ? set_error(MVB_ERR_ARG, "utterance slot %d out of range", utt) : MVB_OK;
}

// ------------------------------------------------------------------------------------------------
// Voices (include/mvb200.h): overlays of blocks [first_layer, n_layer) and ln_f.
extern "C" int mvb_s1_add_voice(mvb_s1* h, const void* d_overlay, size_t overlay_bytes, int32_t first_layer,
                                const uint64_t* offsets, int32_t n_offsets, int32_t* voice) {
  if (!h || !d_overlay || !offsets || !voice) return set_error(MVB_ERR_ARG, "null argument");
  if (h->fmt != WFmt::BF16) return set_error(MVB_ERR_UNSUPPORTED, "voices are served by bf16-weight engines only");
  const mvb_s1_config& c = h->cfg;
  if (first_layer < 0 || first_layer >= c.n_layer)
    return set_error(MVB_ERR_ARG, "first_layer %d outside [0, %d)", first_layer, c.n_layer);
  if ((int)h->voices.size() >= MVB_S1_MAX_VOICES)
    return set_error(MVB_ERR_ARG, "the engine already holds %d voices (MVB_S1_MAX_VOICES)", MVB_S1_MAX_VOICES);
  const bool ln = h->layer_norm(), gelu = h->gelu(), bias = h->arch.bias != 0;
  const int n_w = gelu ? 6 : MVB_S1_LAYER_TENSORS;
  const int n_b = bias ? (ln ? 2 : 0) + 3 + (gelu ? 1 : 2) : 0;
  const int n_ov = c.n_layer - first_layer;
  const int want = n_ov * (n_w + n_b) + 1 + (bias && ln ? 1 : 0);
  if (n_offsets != want)
    return set_error(MVB_ERR_ARG, "an overlay from layer %d has %d tensors, got %d offsets", first_layer, want, n_offsets);
  if (int e = check_offsets(offsets, (size_t)n_offsets, overlay_bytes, "overlay offset")) return e;
  const char* base = reinterpret_cast<const char*>(d_overlay);
  auto at = [&](int i) { return reinterpret_cast<const __nv_bfloat16*>(base + offsets[i]); };
  S1Voice v;
  v.first_layer = first_layer;
  v.t.assign((size_t)n_ov * 7, nullptr);
  v.lp.resize(n_ov);
  v.tmW.resize((size_t)n_ov * 5);
  const int D = c.dim, F = c.intermediate;
  for (int i = 0; i < n_ov; ++i) {
    const int o = i * (n_w + n_b);
    for (int t = 0; t < n_w; ++t) v.t[(size_t)i * 7 + (gelu && t == 5 ? 6 : t)] = at(o + t);
    auto tt = [&](int t) { return v.t[(size_t)i * 7 + t]; };
    S1LayerP& p = v.lp[i];
    p = S1LayerP{};
    p.g1 = tt(0);
    p.g2 = tt(3);
    int nb = o + n_w;                                  // this layer's biases, in mvb_s1_create_ex's order
    auto bias_slot = [&](bool present) { return present && bias ? at(nb++) : nullptr; };
    p.b1 = bias_slot(ln);
    p.qkv_b = bias_slot(true);
    p.o_b = bias_slot(true);
    p.b2 = bias_slot(ln);
    p.fc_b = bias_slot(true);
    p.fc3_b = bias_slot(!gelu);
    p.proj_b = bias_slot(true);
    bool ok = make_tmap_bf16(&v.tmW[(size_t)i * 5 + 0], tt(1), 3 * D, D, 128);
    ok = ok && make_tmap_bf16(&v.tmW[(size_t)i * 5 + 1], tt(2), D, D, 128);
    ok = ok && make_tmap_bf16(&v.tmW[(size_t)i * 5 + 2], tt(4), F, D, 128);
    ok = ok && make_tmap_bf16(&v.tmW[(size_t)i * 5 + 3], tt(gelu ? 4 : 5), F, D, 128);   // GELU: c_fc again
    ok = ok && make_tmap_bf16(&v.tmW[(size_t)i * 5 + 4], tt(6), D, F, 128);
    if (!ok) return set_error(MVB_ERR_CUDA, "cuTensorMapEncodeTiled failed for a matrix of overlay layer %d", first_layer + i);
  }
  const int lf = n_ov * (n_w + n_b);
  v.lnf_g = at(lf);
  v.lnf_b = bias && ln ? at(lf + 1) : nullptr;
  const size_t n_tm = (size_t)c.n_layer * 5 + 1;
  if (!h->vslots) {
    MVB_CK(cudaMalloc(&h->vslots, sizeof(int) * (64 + RB_MAX)));
    h->row_grp = h->vslots + 64;
    MVB_CK(cudaMalloc(&h->vtickets, sizeof(unsigned) * 256 * GEMM_MAX_GROUPS));
    MVB_CK(cudaMemset(h->vtickets, 0, sizeof(unsigned) * 256 * GEMM_MAX_GROUPS));
    MVB_CK(cudaMalloc(&h->d_tm, sizeof(CUtensorMap) * n_tm * MVB_S1_MAX_VOICES));
    MVB_CK(cudaMemcpy(h->d_tm, h->tmW.data(), sizeof(CUtensorMap) * n_tm, cudaMemcpyHostToDevice));
  }
  h->voices.push_back(std::move(v));
  const int id = (int)h->voices.size() - 1;
  std::vector<CUtensorMap> tms(n_tm);
  for (int l = 0; l <= c.n_layer; ++l)
    for (int i = 0; i < (l < c.n_layer ? 5 : 1); ++i) tms[(size_t)l * 5 + i] = *h->vtm(id, l, i);
  MVB_CK(cudaMemcpy(h->d_tm + n_tm * id, tms.data(), sizeof(CUtensorMap) * n_tm, cudaMemcpyHostToDevice));
  *voice = (int32_t)id;
  return MVB_OK;
}

extern "C" int mvb_s1_set_voice(mvb_s1* h, int32_t utt, int32_t voice) {
  if (!h) return set_error(MVB_ERR_ARG, "null handle");
  if (int e = check_slot(h, utt)) return e;
  if (voice < 0 || voice >= (int)h->voices.size())
    return set_error(MVB_ERR_ARG, "voice %d is not registered (%d voices)", voice, (int)h->voices.size());
  h->next_voice[utt] = voice;
  return MVB_OK;
}

extern "C" int mvb_s1_set_speaker(mvb_s1* h, int32_t utt, const float* d_spk, void* stream) {
  if (!h || !d_spk) return set_error(MVB_ERR_ARG, "null argument");
  if (int e = check_slot(h, utt)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  const int D = h->cfg.dim;
  float* out = h->wsp<float>(h->L.spk) + (size_t)utt * D;
  if (h->fmt == WFmt::FP8)
    k_spk_proj<__nv_bfloat16><<<(D * 32 + 255) / 256, 256, 0, s>>>(h->f8_spk, d_spk, out, D, h->cfg.spk_dim,
                                                                    h->tc_scale(2, D, h->cfg.spk_dim));
  else if (h->fmt == WFmt::INT8)
    k_spk_proj<int8_t><<<(D * 32 + 255) / 256, 256, 0, s>>>(reinterpret_cast<const int8_t*>(h->w(2)), d_spk, out, D, h->cfg.spk_dim,
                                                            h->tc_scale(2, D, h->cfg.spk_dim));
  else
    k_spk_proj<__nv_bfloat16><<<(D * 32 + 255) / 256, 256, 0, s>>>(h->w(2), d_spk, out, D, h->cfg.spk_dim, nullptr);
  h->launches++;
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

extern "C" int mvb_s1_forward(mvb_s1* h, int32_t utt, const int32_t* d_idx, int32_t S, int32_t pos0, float* d_logits,
                              int32_t all_positions, void* stream) {
  if (!h || !d_idx) return set_error(MVB_ERR_ARG, "null argument");
  if (int e = check_slot(h, utt)) return e;
  if (S < 1 || pos0 < 0 || pos0 + S > h->cfg.block_size)
    return set_error(MVB_ERR_ARG, "positions [%d, %d) outside the %d-slot context", pos0, pos0 + S, h->cfg.block_size);
  cudaStream_t s = (cudaStream_t)stream;
  const int V = h->cfg.vocab;
  const float* lg = h->wsp<float>(h->L.logits) + (size_t)(2 * utt) * V;
  if (h->path_b && S >= 2) {
    // Prefill on the tensor cores in chunks of PREFILL_CHUNK tokens: every weight matrix is streamed once per
    // chunk for all 2*Sc rows (the reference prefill, utils:123-132, does the same with a [2,T] batch).  Every row is
    // the slot's: it runs with the operands of the slot's voice.
    const mvb_s1_config& c = h->cfg;
    const int voice = h->slot_voice[utt];
    for (int s0 = 0; s0 < S; s0 += PREFILL_CHUNK) {
      const int Sc = (S - s0) < PREFILL_CHUNK ? (S - s0) : PREFILL_CHUNK;
      const int R = 2 * Sc;
      k_rows_prefill<<<1, 128, 0, s>>>(h->rows, utt, d_idx, S, s0, Sc, pos0);
      h->launches++;
      MVB_CK(cudaGetLastError());
      if (int e = launch_layers_b(h, s, R, voice)) return e;
      float* bx = h->wsp<float>(h->L.b_x);
      if (d_logits && all_positions) {
        float* bl = h->wsp<float>(h->L.b_logits);
        if (int e = head_b(h, s, R, bx, bl, voice)) return e;
        for (int cc = 0; cc < 2; ++cc)
          MVB_CK(cudaMemcpyAsync(d_logits + ((size_t)cc * S + s0) * V, bl + (size_t)cc * Sc * V, sizeof(float) * (size_t)Sc * V,
                             cudaMemcpyDeviceToDevice, s));
      }
      if (s0 + Sc == S) {
        // last position -> the sampler's logits rows of this utterance (and the decode state's position)
        float* last = h->wsp<float>(h->L.b_last);
        k_gather_last<<<2, 256, 0, s>>>(bx, last, Sc, c.dim);
        h->launches++;
        MVB_CK(cudaGetLastError());
        if (int e = head_b(h, s, 2, last, h->wsp<float>(h->L.logits) + (size_t)(2 * utt) * V, voice)) return e;
        k_set_input<<<1, 32, 0, s>>>(h->st, utt, d_idx, S, S - 1, pos0 + S - 1);
        h->launches++;
        MVB_CK(cudaGetLastError());
      }
    }
    if (d_logits && !all_positions) MVB_CK(cudaMemcpyAsync(d_logits, lg, sizeof(float) * 2 * V, cudaMemcpyDeviceToDevice, s));
    return MVB_OK;
  }
  for (int i = 0; i < S; ++i) {
    k_set_input<<<1, 32, 0, s>>>(h->st, utt, d_idx, S, i, pos0 + i);
    h->launches++;
    MVB_CK(cudaGetLastError());
    if (int e = run_body(h, s, 1, false, utt)) return e;
    if (d_logits && all_positions) {
      MVB_CK(cudaMemcpyAsync(d_logits + (size_t)i * V, lg, sizeof(float) * V, cudaMemcpyDeviceToDevice, s));
      MVB_CK(cudaMemcpyAsync(d_logits + ((size_t)S + i) * V, lg + V, sizeof(float) * V, cudaMemcpyDeviceToDevice, s));
    }
  }
  if (d_logits && !all_positions) MVB_CK(cudaMemcpyAsync(d_logits, lg, sizeof(float) * 2 * V, cudaMemcpyDeviceToDevice, s));
  return MVB_OK;
}

// k_sample in API mode; prompt_guidance > 1 mixes the three rows of d_logits [3, V], anything else the two of [2, V].
static int sample_api(mvb_s1* h, const float* d_logits, const mvb_sampling* p, float prompt_guidance, const float* d_noise,
                      uint64_t step, int32_t* d_token_out, float* d_probs_out, void* stream) {
  SampleP sp{};
  sp.logits = d_logits;
  sp.V = h->cfg.vocab;
  sp.decode_mode = 0;
  sp.sp = to_dev(p);
  sp.prompt_guidance = prompt_guidance;
  sp.noise = d_noise;
  sp.step = step;
  sp.token_out = d_token_out;
  sp.probs_out = d_probs_out;
  k_sample<<<1, SAMP_THREADS, 0, (cudaStream_t)stream>>>(sp, h->st);
  h->launches++;
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

extern "C" int mvb_s1_sample(mvb_s1* h, const float* d_logits, const mvb_sampling* p, const float* d_noise, uint64_t step,
                             int32_t* d_token_out, float* d_probs_out, void* stream) {
  if (!h || !d_logits || !p || !d_token_out) return set_error(MVB_ERR_ARG, "null argument");
  return sample_api(h, d_logits, p, 1.0f, d_noise, step, d_token_out, d_probs_out, stream);
}

// The reference asserts both guidance scales (causal.py:87-88): finite and >= 1.
static int check_guidance(float s, float pg) {
  if (!std::isfinite(s) || !std::isfinite(pg) || s < 1.0f || pg < 1.0f)
    return set_error(MVB_ERR_ARG, "guidance_scale (%g, %g): both scales must be finite and >= 1", (double)s, (double)pg);
  return MVB_OK;
}

extern "C" int mvb_s1_sample_guided(mvb_s1* h, const float* d_logits, const mvb_sampling* p, float prompt_guidance_scale,
                                    const float* d_noise, uint64_t step, int32_t* d_token_out, float* d_probs_out, void* stream) {
  if (!h || !d_logits || !p || !d_token_out) return set_error(MVB_ERR_ARG, "null argument");
  if (int e = check_guidance(p->guidance_scale, prompt_guidance_scale)) return e;
  return sample_api(h, d_logits, p, prompt_guidance_scale, d_noise, step, d_token_out, d_probs_out, stream);
}

// Prompt-guidance link of a primary u and its companion c (SamplingDev::link); the companion's entry takes p and
// end_of_text.  k_unlink dissolves a link on both sides and parks the former companion.
__global__ void k_link(S1State st, int u, int c, float prompt_guidance, int end_of_text) {
  if (threadIdx.x == 0) {
    st.samp[u].link = c + 1;
    st.samp[c].link = -(u + 1);
    st.samp[c].guidance = prompt_guidance;
    st.samp[c].end_of_audio = end_of_text;
  }
}
__global__ void k_unlink(S1State st, int a, int b, int companion) {
  if (threadIdx.x == 0) {
    st.samp[a].link = 0;
    st.samp[b].link = 0;
    st.done[companion] = 1;
  }
}

static int unlink_slot(mvb_s1* h, int utt, cudaStream_t s) {
  const int l = h->h_link[utt];
  if (l == 0) return MVB_OK;
  const int partner = l > 0 ? l - 1 : -l - 1;
  k_unlink<<<1, 32, 0, s>>>(h->st, utt, partner, l > 0 ? partner : utt);
  h->launches++;
  MVB_CK(cudaGetLastError());
  h->h_link[utt] = h->h_link[partner] = 0;
  return MVB_OK;
}

extern "C" int mvb_s1_begin(mvb_s1* h, int32_t utt, int32_t first_token, int32_t pos, const mvb_sampling* p,
                            const float* d_noise, const int32_t* d_forced, void* stream) {
  if (!h || !p) return set_error(MVB_ERR_ARG, "null argument");
  if (int e = check_slot(h, utt)) return e;
  if (pos < 0 || pos >= h->cfg.block_size) return set_error(MVB_ERR_ARG, "position %d outside the context", pos);
  if (int e = unlink_slot(h, utt, (cudaStream_t)stream)) return e;
  h->h_topk[utt] = p->top_k;
  h->slot_voice[utt] = h->next_voice[utt];
  k_begin<<<1, 32, 0, (cudaStream_t)stream>>>(h->st, utt, first_token, pos, to_dev(p), d_noise, d_forced, first_token >= 0,
                                              h->cfg.max_new);
  h->launches++;
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

// per-utterance token budget (generate(): utils:196-204) and the step that row 0 of the staged noise belongs to
__global__ void k_set_budget(S1State st, int utt, int budget) {
  if (threadIdx.x == 0) st.budget[utt] = budget;
}
__global__ void k_set_noise_base(S1State st, int n_utts, int base) {
  if ((int)threadIdx.x < n_utts) st.noise_base[threadIdx.x] = base;
}
__global__ void k_set_done(S1State st, int utt, int done) {
  if (threadIdx.x == 0) st.done[utt] = done;
}

// ------------------------------------------------------------------------------------------------
// Continuous batching (SURVEY.md row N4): utterances enter and leave KV slots between decode bursts.
// mvb_s1_admit == the per-utterance prologue of generate() (utils:196-212): budget check, prompt / speaker upload,
// prefill, first token sampled from the last prompt position.  The slot then rides along in every mvb_s1_decode burst
// until its done flag latches (mvb_s1_poll), after which the host fetches its tokens and may admit another request.
// Argument checks of an admission: the prompt length and token budget (generate(): utils:196-204) -> *room.
static int admit_room(const mvb_s1* h, int32_t T, int32_t max_new_tokens, int* room) {
  const mvb_s1_config& c = h->cfg;
  if (T < 1) return set_error(MVB_ERR_ARG, "empty prompt");
  if (max_new_tokens < 1 || max_new_tokens > c.max_new) return set_error(MVB_ERR_ARG, "max_new_tokens %d out of range", max_new_tokens);
  *room = (T + max_new_tokens < c.block_size ? T + max_new_tokens : c.block_size) - T;
  if (*room <= 0) return set_error(MVB_ERR_PROMPT_TOO_LONG, "Prompt is too long to generate more tokens");
  return MVB_OK;
}

// Prompt / speaker upload, decode state and prefill of slot `utt` on voice `voice`: everything of an admission but the
// first sample.
static int admit_prefill(mvb_s1* h, int32_t utt, const int32_t* prompt, int32_t T, const float* spk_emb,
                         const mvb_sampling* params, int room, const float* d_noise, int voice, cudaStream_t s) {
  const mvb_s1_config& c = h->cfg;
  int* di = h->wsp<int>(h->L.stage_idx) + (size_t)utt * 2 * c.block_size;
  float* d_spk = h->wsp<float>(h->L.stage_spk) + (size_t)utt * c.spk_dim;
  MVB_CK(cudaMemcpyAsync(d_spk, spk_emb, sizeof(float) * c.spk_dim, cudaMemcpyHostToDevice, s));
  MVB_CK(cudaMemcpyAsync(di, prompt, sizeof(int) * T, cudaMemcpyHostToDevice, s));
  MVB_CK(cudaMemcpyAsync(di + T, prompt, sizeof(int) * T, cudaMemcpyHostToDevice, s));
  if (int e = mvb_s1_set_speaker(h, utt, d_spk, s)) return e;
  if (int e = mvb_s1_begin(h, utt, -1, 0, params, d_noise, nullptr, s)) return e;
  h->slot_voice[utt] = voice;
  k_set_budget<<<1, 32, 0, s>>>(h->st, utt, room);
  h->launches++;
  return mvb_s1_forward(h, utt, di, T, 0, nullptr, 0, s);
}

// The first token of the slot prefilled last (slot_map[0] == that slot after the prefill), in decode mode.
static int admit_sample(mvb_s1* h, cudaStream_t s) {
  SampleP spp{};
  spp.logits = h->wsp<float>(h->L.logits);
  spp.V = h->cfg.vocab;
  spp.decode_mode = 1;
  k_sample<<<1, SAMP_THREADS, 0, s>>>(spp, h->st);
  h->launches++;
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

extern "C" int mvb_s1_admit(mvb_s1* h, int32_t utt, const int32_t* prompt, int32_t T, const float* spk_emb,
                            const mvb_sampling* params, int32_t max_new_tokens, const float* d_noise, void* stream) {
  if (!h || !prompt || !spk_emb || !params) return set_error(MVB_ERR_ARG, "null argument");
  if (int e = check_slot(h, utt)) return e;
  int room = 0;
  if (int e = admit_room(h, T, max_new_tokens, &room)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  if (int e = admit_prefill(h, utt, prompt, T, spk_emb, params, room, d_noise, h->next_voice[utt], s)) return e;
  return admit_sample(h, s);
}

// Prompt guidance (_sample_batch with guidance_scale = (s, p), causal.py:224-262): the companion slot is prefilled with
// the prompt's text tokens replaced by end_of_text under the same speaker, the primary as mvb_s1_admit does, then the
// link is installed and the first token is sampled from the three rows.  p == 1 is mvb_s1_admit: no companion.
extern "C" int mvb_s1_admit_guided(mvb_s1* h, int32_t utt, int32_t companion, const int32_t* prompt, int32_t T,
                                   const float* spk_emb, const mvb_sampling* params, float prompt_guidance_scale,
                                   int32_t end_of_text_token, int32_t max_new_tokens, const float* d_noise, void* stream) {
  if (!h || !prompt || !spk_emb || !params) return set_error(MVB_ERR_ARG, "null argument");
  if (int e = check_slot(h, utt)) return e;
  if (int e = check_slot(h, companion)) return e;
  if (companion == utt) return set_error(MVB_ERR_ARG, "companion slot %d is the utterance's own slot", companion);
  if (int e = check_guidance(params->guidance_scale, prompt_guidance_scale)) return e;
  if (end_of_text_token < 0 || end_of_text_token >= h->cfg.vocab)
    return set_error(MVB_ERR_ARG, "end_of_text_token %d outside the vocabulary", end_of_text_token);
  int room = 0;
  if (int e = admit_room(h, T, max_new_tokens, &room)) return e;
  if (prompt_guidance_scale == 1.0f) return mvb_s1_admit(h, utt, prompt, T, spk_emb, params, max_new_tokens, d_noise, stream);
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<int32_t> uncond(prompt, prompt + T);   // causal.py:259-262
  for (int32_t& t : uncond)
    if (t > params->end_of_audio) t = end_of_text_token;
  // the uncond-prompt row runs through the primary's model: the companion takes the primary's voice
  if (int e = admit_prefill(h, companion, uncond.data(), T, spk_emb, params, room, nullptr, h->next_voice[utt], s)) return e;
  if (int e = admit_prefill(h, utt, prompt, T, spk_emb, params, room, d_noise, h->next_voice[utt], s)) return e;
  k_link<<<1, 32, 0, s>>>(h->st, utt, companion, prompt_guidance_scale, end_of_text_token);
  h->launches++;
  MVB_CK(cudaGetLastError());
  h->h_link[utt] = companion + 1;
  h->h_link[companion] = -(utt + 1);
  return admit_sample(h, s);
}

// A parked or finished slot (and a guided primary's companion) goes back to voice 0: its rows still ride along in the
// batch, and must not keep a batch of live voice-0 slots off the resident decode kernel or stream an overlay for it.
static void park_voice(mvb_s1* h, int utt) {
  h->slot_voice[utt] = 0;
  const int l = h->h_link[utt];
  if (l > 0) h->slot_voice[l - 1] = 0;
}

// Park a slot: its rows still ride along in the batch (recomputed at a frozen position) but nothing is sampled or
// appended for it until the next mvb_s1_admit / mvb_s1_begin.
extern "C" int mvb_s1_release(mvb_s1* h, int32_t utt, void* stream) {
  if (!h) return set_error(MVB_ERR_ARG, "null handle");
  if (int e = check_slot(h, utt)) return e;
  k_set_done<<<1, 32, 0, (cudaStream_t)stream>>>(h->st, utt, 1);
  h->launches++;
  MVB_CK(cudaGetLastError());
  park_voice(h, utt);
  if (h->h_link[utt] > 0) return unlink_slot(h, utt, (cudaStream_t)stream);   // a guided primary parks its companion too
  return MVB_OK;
}

// A guided primary whose done flag the host has read has finished for good (only an admission or mvb_s1_begin clears the
// flag): its link is dissolved here, so that later bursts may leave the old companion out and sample unguided slots in
// the resident kernel again.
static int unlink_finished(mvb_s1* h, int32_t utt, int done, cudaStream_t s) {
  if (done) park_voice(h, utt);
  return (done && h->h_link[utt] > 0) ? unlink_slot(h, utt, s) : MVB_OK;
}

// done flags and generated-token counts of slots [0, n_slots) in one device->host round trip (synchronises `stream`).
extern "C" int mvb_s1_poll(mvb_s1* h, int32_t n_slots, int32_t* done_out, int32_t* n_gen_out, void* stream) {
  if (!h || !done_out || !n_gen_out) return set_error(MVB_ERR_ARG, "null argument");
  if (n_slots < 1 || n_slots > h->cfg.max_utts) return set_error(MVB_ERR_ARG, "n_slots %d out of range", n_slots);
  cudaStream_t s = (cudaStream_t)stream;
  MVB_CK(cudaMemcpyAsync(h->h_flags, h->st.done, sizeof(int) * n_slots, cudaMemcpyDeviceToHost, s));
  MVB_CK(cudaMemcpyAsync(h->h_flags + 64, h->st.n_gen, sizeof(int) * n_slots, cudaMemcpyDeviceToHost, s));
  MVB_CK(cudaStreamSynchronize(s));
  for (int i = 0; i < n_slots; ++i) { done_out[i] = h->h_flags[i]; n_gen_out[i] = h->h_flags[64 + i]; }
  for (int i = 0; i < n_slots; ++i)
    if (int e = unlink_finished(h, i, done_out[i], s)) return e;
  return MVB_OK;
}

static int sample_step(mvb_s1* h, cudaStream_t s, int n_utts) {
  SampleP sp{};
  sp.logits = h->wsp<float>(h->L.logits);
  sp.V = h->cfg.vocab;
  sp.decode_mode = 1;
  sp.grid_bar = h->wsp<unsigned>(h->L.c_bar);
  h->launches++;
  MVB_CK(launch_pdl(k_sample, dim3(n_utts), dim3(SAMP_THREADS), 0, s, sp, h->st));
  return MVB_OK;
}

extern "C" int mvb_s1_decode(mvb_s1* h, int32_t n_utts, int32_t n_steps, void* stream) {
  if (!h) return set_error(MVB_ERR_ARG, "null handle");
  if (n_utts < 1 || n_utts > h->cfg.max_utts) return set_error(MVB_ERR_ARG, "n_utts %d out of range", n_utts);
  for (int u = 0; u < n_utts; ++u) {   // a guided primary samples from its companion's rows: both must be decoded
    const int l = h->h_link[u], partner = l > 0 ? l - 1 : -l - 1;
    if (l != 0 && partner >= n_utts)
      return set_error(MVB_ERR_ARG, "slot %d is linked to slot %d outside the %d decoded slots", u, partner, n_utts);
  }
  if (n_steps < 1) return MVB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  k_identity_slots<<<1, 64, 0, s>>>(h->st, n_utts);
  h->launches++;
  MVB_CK(cudaGetLastError());
  const bool use_c = use_path_c(h, n_utts);
  if (use_c) {
    // The persistent kernel ACCUMULATES split-K partial logits (red.add); a prefill (mvb_s1_forward) leaves the last
    // position's logits in the same rows, so they must be zero before the first fused step.  Its grid-barrier counter
    // starts from zero at every launch.
    MVB_CK(cudaMemsetAsync(h->wsp<float>(h->L.logits), 0, sizeof(float) * 2 * (size_t)n_utts * h->cfg.vocab, s));
    // One launch for the whole burst: the kernel samples on the device (top_k = None only, the stage-1 default of
    // TTS.synthesise) and stays resident across positions.
    bool fused = h->fused && (h->cfg.vocab + h->n_sm - 1) / h->n_sm <= PC_SAMP_OWN && h->cfg.vocab <= SAMP_PAD;
    for (int u = 0; u < n_utts; ++u) fused = fused && h->h_topk[u] <= 0 && h->h_link[u] == 0;   // top-k and guided: k_sample
    if (fused) return launch_persistent(h, s, n_utts, n_steps, true);
  }
  for (int i = 0; i < n_steps; ++i) {
    if (use_c) {
      if (int e = launch_persistent(h, s, n_utts, 1, false)) return e;   // (the sampler below resets the barrier counter)
    } else {
      if (int e = run_body(h, s, n_utts)) return e;
    }
    if (int e = sample_step(h, s, n_utts)) return e;
  }
  return MVB_OK;
}


// Parity hook for the decode body: one position for utterances [0, n_utts) from the current decode state (tokens /
// positions installed with mvb_s1_begin) through the body mvb_s1_decode runs for that batch, logits copied out, no
// sampling, state untouched except for the KV-cache append at the current positions.  That body is the persistent
// fused kernel where mvb_s1_decode would use it (up to 8 utterances), else the per-layer path (tensor-core rows path
// from 2 utterances up).
extern "C" int mvb_s1_step_logits(mvb_s1* h, int32_t n_utts, float* d_logits, void* stream) {
  if (!h || !d_logits) return set_error(MVB_ERR_ARG, "null argument");
  if (n_utts < 1 || n_utts > h->cfg.max_utts) return set_error(MVB_ERR_ARG, "n_utts %d out of range", n_utts);
  cudaStream_t s = (cudaStream_t)stream;
  const size_t bytes = sizeof(float) * 2 * (size_t)n_utts * h->cfg.vocab;
  k_identity_slots<<<1, 64, 0, s>>>(h->st, n_utts);
  h->launches++;
  MVB_CK(cudaGetLastError());
  if (!use_path_c(h, n_utts)) {
    if (int e = run_body(h, s, n_utts)) return e;
    MVB_CK(cudaMemcpyAsync(d_logits, h->wsp<float>(h->L.logits), bytes, cudaMemcpyDeviceToDevice, s));
    return MVB_OK;
  }
  MVB_CK(cudaMemsetAsync(h->wsp<float>(h->L.logits), 0, bytes, s));
  MVB_CK(cudaMemsetAsync(h->wsp<unsigned>(h->L.c_bar), 0, 4, s));
  if (int e = launch_persistent(h, s, n_utts, 1, false)) return e;
  MVB_CK(cudaMemcpyAsync(d_logits, h->wsp<float>(h->L.logits), bytes, cudaMemcpyDeviceToDevice, s));
  MVB_CK(cudaMemsetAsync(h->wsp<float>(h->L.logits), 0, bytes, s));
  MVB_CK(cudaMemsetAsync(h->wsp<unsigned>(h->L.c_bar), 0, 4, s));
  return MVB_OK;
}

// Debug: copy the persistent kernel's per-CTA phase time stamps (clock64) of the last step to the host.
extern "C" int mvb_s1_trace_fetch(mvb_s1* h, long long* out, int32_t max_ctas, void* stream) {
  if (!h || !out) return set_error(MVB_ERR_ARG, "null argument");
  const int n = h->n_sm < max_ctas ? h->n_sm : max_ctas;
  MVB_CK(cudaMemcpyAsync(out, h->wsp<long long>(h->L.c_trace), sizeof(long long) * (size_t)n * PC_TRACE_EVENTS, cudaMemcpyDeviceToHost,
                     (cudaStream_t)stream));
  MVB_CK(cudaStreamSynchronize((cudaStream_t)stream));
  return n;
}

extern "C" int mvb_s1_fetch(mvb_s1* h, int32_t utt, int32_t* out_tokens, int32_t cap, int32_t* n_out, int32_t* done,
                            void* stream) {
  if (!h) return set_error(MVB_ERR_ARG, "null handle");
  if (int e = check_slot(h, utt)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  MVB_CK(cudaMemcpyAsync(h->h_flags, h->st.n_gen + utt, 4, cudaMemcpyDeviceToHost, s));
  MVB_CK(cudaMemcpyAsync(h->h_flags + 1, h->st.done + utt, 4, cudaMemcpyDeviceToHost, s));
  MVB_CK(cudaStreamSynchronize(s));
  const int n = h->h_flags[0], finished = h->h_flags[1];
  if (n_out) *n_out = n;
  if (done) *done = finished;
  if (out_tokens && cap > 0) {
    const int m = n < cap ? n : cap;
    MVB_CK(cudaMemcpyAsync(out_tokens, h->st.gen_tokens + (size_t)utt * h->cfg.max_new, sizeof(int) * m, cudaMemcpyDeviceToHost, s));
    MVB_CK(cudaStreamSynchronize(s));
  }
  return unlink_finished(h, utt, finished, s);
}

// Sampled (pre-teacher-forcing) tokens, for the parity tests.
extern "C" int mvb_s1_fetch_sampled(mvb_s1* h, int32_t utt, int32_t* out_tokens, int32_t cap, void* stream) {
  if (!h || !out_tokens) return set_error(MVB_ERR_ARG, "null argument");
  if (int e = check_slot(h, utt)) return e;
  if (cap < 0 || cap > h->cfg.max_new) return set_error(MVB_ERR_ARG, "cap %d outside [0, %d]", cap, h->cfg.max_new);
  cudaStream_t s = (cudaStream_t)stream;
  MVB_CK(cudaMemcpyAsync(out_tokens, h->st.sampled_tokens + (size_t)utt * h->cfg.max_new, sizeof(int) * cap, cudaMemcpyDeviceToHost, s));
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}

extern "C" int mvb_s1_generate(mvb_s1* h, int32_t n_utts, const int32_t* prompts, const int32_t* prompt_lens,
                               const float* spk_embs, const mvb_sampling* params, int32_t max_new_tokens,
                               const float* noise, int32_t noise_on_device, const int32_t* forced, int32_t* out_tokens,
                               int32_t* out_lens, void* stream) {
  if (!h || !prompts || !prompt_lens || !spk_embs || !params || !out_tokens || !out_lens)
    return set_error(MVB_ERR_ARG, "null argument");
  const mvb_s1_config& c = h->cfg;
  if (n_utts < 1 || n_utts > c.max_utts) return set_error(MVB_ERR_ARG, "n_utts %d exceeds the %d slots", n_utts, c.max_utts);
  if (max_new_tokens < 1 || max_new_tokens > c.max_new) return set_error(MVB_ERR_ARG, "max_new_tokens %d out of range", max_new_tokens);
  cudaStream_t s = (cudaStream_t)stream;
  // generate(): max_seq = min(T + max_new, block_size); raise if no room (utils:196-204)
  std::vector<int> budget(n_utts);
  for (int i = 0; i < n_utts; ++i) {
    const int T = prompt_lens[i];
    if (T < 1) return set_error(MVB_ERR_ARG, "empty prompt for utterance %d", i);
    const int room = (T + max_new_tokens < c.block_size ? T + max_new_tokens : c.block_size) - T;
    if (room <= 0) return set_error(MVB_ERR_PROMPT_TOO_LONG, "Prompt is too long to generate more tokens");
    budget[i] = room;
  }
  const int V = c.vocab;
  // Exp(1) draws: a device buffer is used in place; a host buffer is staged one burst of decode steps at a time
  // into the workspace (no allocation inside the call).
  const bool stage_noise = noise != nullptr && !noise_on_device;
  float* d_stage = h->wsp<float>(h->L.stage_noise);
  auto stage_rows = [&](int step0, int rows) -> int {
    for (int i = 0; i < n_utts; ++i)
      MVB_CK(cudaMemcpyAsync(d_stage + (size_t)i * GEN_BURST * V, noise + ((size_t)i * max_new_tokens + step0) * V,
                         sizeof(float) * (size_t)rows * V, cudaMemcpyHostToDevice, s));
    k_set_noise_base<<<1, 64, 0, s>>>(h->st, n_utts, step0);
    h->launches++;
    MVB_CK(cudaGetLastError());
    return MVB_OK;
  };
  int* d_forced = h->wsp<int>(h->L.stage_forced);
  if (forced) MVB_CK(cudaMemcpyAsync(d_forced, forced, sizeof(int) * (size_t)n_utts * max_new_tokens, cudaMemcpyHostToDevice, s));
  int* d_idx = h->wsp<int>(h->L.stage_idx);
  float* d_spk = h->wsp<float>(h->L.stage_spk);
  MVB_CK(cudaMemcpyAsync(d_spk, spk_embs, sizeof(float) * (size_t)n_utts * c.spk_dim, cudaMemcpyHostToDevice, s));
  int rc = MVB_OK;
  size_t poff = 0;
  int max_budget = 0;
  for (int i = 0; i < n_utts && rc == MVB_OK; ++i) {
    const int T = prompt_lens[i];
    int* di = d_idx + (size_t)i * 2 * c.block_size;
    // prompt.view(1,-1).repeat(2,1): both CFG rows see the same tokens (utils:211)
    MVB_CK(cudaMemcpyAsync(di, prompts + poff, sizeof(int) * T, cudaMemcpyHostToDevice, s));
    MVB_CK(cudaMemcpyAsync(di + T, prompts + poff, sizeof(int) * T, cudaMemcpyHostToDevice, s));
    poff += T;
    if ((rc = mvb_s1_set_speaker(h, i, d_spk + (size_t)i * c.spk_dim, s))) break;
    mvb_sampling sp = params[i];
    const float* dn = nullptr;
    if (stage_noise) dn = d_stage + (size_t)i * GEN_BURST * V;
    else if (noise) dn = noise + (size_t)i * max_new_tokens * V;
    if ((rc = mvb_s1_begin(h, i, -1, 0, &sp, dn, forced ? d_forced + (size_t)i * max_new_tokens : nullptr, s))) break;
    k_set_budget<<<1, 32, 0, s>>>(h->st, i, budget[i]);
    h->launches++;
    if (budget[i] > max_budget) max_budget = budget[i];
  }
  if (rc == MVB_OK && stage_noise) rc = stage_rows(0, 1);      // row 0 feeds the post-prefill samples below
  for (int i = 0; i < n_utts && rc == MVB_OK; ++i) {
    const int T = prompt_lens[i];
    int* di = d_idx + (size_t)i * 2 * c.block_size;
    if ((rc = mvb_s1_forward(h, i, di, T, 0, nullptr, 0, s))) break;  // prefill (utils:123-132)
    // first token sampled from the last prefill position (utils:211-212)
    SampleP spp{};
    spp.logits = h->wsp<float>(h->L.logits);
    spp.V = V;
    spp.decode_mode = 1;
    k_sample<<<1, SAMP_THREADS, 0, s>>>(spp, h->st);  // slot_map[0] == i after the prefill
    h->launches++;
    if (cudaGetLastError() != cudaSuccess) { rc = set_error(MVB_ERR_CUDA, "sampler launch failed"); break; }
  }
  // decode_n_tokens: at most budget-1 further steps, all utterances advance together with their own positions;
  // per-utterance budgets and the end of the context are latched on the device (done flag).
  if (rc == MVB_OK) {
    int remaining = max_budget - 1, step0 = 1;
    while (remaining > 0 && rc == MVB_OK) {
      const int burst = remaining < GEN_BURST ? remaining : GEN_BURST;
      if (stage_noise && (rc = stage_rows(step0, burst))) break;
      rc = mvb_s1_decode(h, n_utts, burst, s);
      remaining -= burst;
      step0 += burst;
      if (rc) break;
      MVB_CK(cudaMemcpyAsync(h->h_flags, h->st.done, sizeof(int) * n_utts, cudaMemcpyDeviceToHost, s));
      MVB_CK(cudaStreamSynchronize(s));
      bool all = true;
      for (int i = 0; i < n_utts; ++i) all = all && h->h_flags[i];
      if (all) break;
    }
  }
  if (rc == MVB_OK) {
    MVB_CK(cudaMemcpyAsync(h->h_flags, h->st.n_gen, sizeof(int) * n_utts, cudaMemcpyDeviceToHost, s));
    MVB_CK(cudaStreamSynchronize(s));
    for (int i = 0; i < n_utts; ++i) {
      int n = h->h_flags[i];
      if (n > budget[i]) n = budget[i];
      out_lens[i] = n;
      MVB_CK(cudaMemcpyAsync(out_tokens + (size_t)i * max_new_tokens, h->st.gen_tokens + (size_t)i * c.max_new, sizeof(int) * n,
                         cudaMemcpyDeviceToHost, s));
    }
    MVB_CK(cudaStreamSynchronize(s));
  }
  return rc;
}

// ------------------------------------------------------------------------------------------------
// Test hooks of the path-A GEMVs (include/mvb200.h): k_gemv / k_gemv_w4 / k_gemv_w8 / k_gemv_f8 with epilogue epi exactly
// as path A launches them, over a caller-built decode state (slot map and positions).  The caller checks the arguments.
static int gemv_test(WFmt fmt, int32_t epi, bool layer, const void* d_W, const void* d_W3, const void* d_bias,
                     const void* d_bias3, int32_t M, int32_t K, const float* d_x, int32_t ldx, int32_t n_utts,
                     const void* d_gain, const void* d_beta, float eps, float* d_out, int32_t ldo, void* d_kcache,
                     void* d_vcache, const int32_t* d_slot_map, const int32_t* d_pos, int32_t H, int32_t S_max, int32_t D,
                     int32_t kv_fp32, cudaStream_t s) {
  mvb_s1 h{};
  int dev = 0;
  if (int e = current_device(&dev, &h.n_sm)) return e;
  h.st.slot_map = const_cast<int*>(d_slot_map);
  h.st.pos = const_cast<int*>(d_pos);
  GemvP p{};
  p.W = reinterpret_cast<const __nv_bfloat16*>(d_W); p.W3 = reinterpret_cast<const __nv_bfloat16*>(d_W3);
  p.x = d_x; p.ldx = ldx; p.gain = reinterpret_cast<const __nv_bfloat16*>(d_gain); p.eps = eps;
  p.beta = reinterpret_cast<const __nv_bfloat16*>(d_beta);
  p.bias = reinterpret_cast<const __nv_bfloat16*>(d_bias);
  p.bias3 = epi == EPI_SWIGLU ? reinterpret_cast<const __nv_bfloat16*>(d_bias3) : nullptr;
  p.out = d_out; p.ldo = ldo; p.M = M; p.K = K;
  p.kcache = d_kcache; p.vcache = d_vcache; p.H = H; p.S_max = S_max; p.D = D; p.kv_fp32 = kv_fp32;
  switch (epi) {
    case EPI_STORE: MVB_CK(launch_gemv<EPI_STORE>(&h, s, n_utts, p, fmt, layer)); break;
    case EPI_RESID: MVB_CK(launch_gemv<EPI_RESID>(&h, s, n_utts, p, fmt, layer)); break;
    case EPI_SWIGLU: MVB_CK(launch_gemv<EPI_SWIGLU>(&h, s, n_utts, p, fmt, layer)); break;
    case EPI_QKV: MVB_CK(launch_gemv<EPI_QKV>(&h, s, n_utts, p, fmt, layer)); break;
    default: MVB_CK(launch_gemv<EPI_GELU>(&h, s, n_utts, p, fmt, layer)); break;
  }
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}

// The int4, int8 and fp8 GEMVs.
static int quant_gemv_test(WFmt fmt, int32_t epi, const void* d_W, const void* d_W3, int32_t M, int32_t K, const float* d_x,
                           int32_t ldx, int32_t n_utts, const void* d_gain, float eps, float* d_out, int32_t ldo,
                           void* d_kcache, void* d_vcache, const int32_t* d_slot_map, const int32_t* d_pos, int32_t H,
                           int32_t S_max, int32_t D, int32_t kv_fp32, void* stream) {
  if (!d_W || !d_x || !d_out || !d_slot_map || !d_pos) return set_error(MVB_ERR_ARG, "null argument");
  if (epi < EPI_STORE || epi > EPI_QKV) return set_error(MVB_ERR_ARG, "bad epilogue %d", epi);
  if (K < 256 || K % 256 || M < 2 || M % 2 || n_utts < 1 || n_utts > 64) return set_error(MVB_ERR_ARG, "bad shape M=%d K=%d n_utts=%d", M, K, n_utts);
  if (fmt != WFmt::FP8 && (size_t)2 * K * sizeof(float) > 48 * 1024)
    return set_error(MVB_ERR_UNSUPPORTED, "K=%d exceeds the staging buffer", K);
  if (fmt == WFmt::FP8 && ldx % 2) return set_error(MVB_ERR_ARG, "ldx=%d must be even", ldx);
  if (epi == EPI_SWIGLU && !d_W3) return set_error(MVB_ERR_ARG, "SwiGLU needs W3");
  if (epi == EPI_QKV && (!d_kcache || !d_vcache || M != 3 * D || D != 128 * H)) return set_error(MVB_ERR_ARG, "bad QKV arguments");
  return gemv_test(fmt, epi, false, d_W, d_W3, nullptr, nullptr, M, K, d_x, ldx, n_utts, d_gain, nullptr, eps, d_out, ldo,
                   d_kcache, d_vcache, d_slot_map, d_pos, H, S_max, D, kv_fp32, (cudaStream_t)stream);
}

extern "C" int mvb_w4_gemv_test(int32_t epi, const void* d_W, const void* d_W3, int32_t M, int32_t K, const float* d_x,
                                int32_t ldx, int32_t n_utts, const void* d_gain, float eps, float* d_out, int32_t ldo,
                                void* d_kcache, void* d_vcache, const int32_t* d_slot_map, const int32_t* d_pos, int32_t H,
                                int32_t S_max, int32_t D, int32_t kv_fp32, void* stream) {
  return quant_gemv_test(WFmt::INT4, epi, d_W, d_W3, M, K, d_x, ldx, n_utts, d_gain, eps, d_out, ldo, d_kcache, d_vcache,
                         d_slot_map, d_pos, H, S_max, D, kv_fp32, stream);
}

extern "C" int mvb_w8_gemv_test(int32_t epi, const void* d_W, const void* d_W3, int32_t M, int32_t K, const float* d_x,
                                int32_t ldx, int32_t n_utts, const void* d_gain, float eps, float* d_out, int32_t ldo,
                                void* d_kcache, void* d_vcache, const int32_t* d_slot_map, const int32_t* d_pos, int32_t H,
                                int32_t S_max, int32_t D, int32_t kv_fp32, void* stream) {
  return quant_gemv_test(WFmt::INT8, epi, d_W, d_W3, M, K, d_x, ldx, n_utts, d_gain, eps, d_out, ldo, d_kcache, d_vcache,
                         d_slot_map, d_pos, H, S_max, D, kv_fp32, stream);
}

extern "C" int mvb_f8_gemv_test(int32_t epi, const void* d_W, const void* d_W3, int32_t M, int32_t K, const float* d_x,
                                int32_t ldx, int32_t n_utts, const void* d_gain, float eps, float* d_out, int32_t ldo,
                                void* d_kcache, void* d_vcache, const int32_t* d_slot_map, const int32_t* d_pos, int32_t H,
                                int32_t S_max, int32_t D, int32_t kv_fp32, void* stream) {
  return quant_gemv_test(WFmt::FP8, epi, d_W, d_W3, M, K, d_x, ldx, n_utts, d_gain, eps, d_out, ldo, d_kcache, d_vcache,
                         d_slot_map, d_pos, H, S_max, D, kv_fp32, stream);
}

// k_w4_dequant / k_w8_widen / k_f8_widen on one matrix (an fp8 matrix has an even M).
static int widen_test(WFmt fmt, const void* d_W, int32_t M, int32_t K, void* d_out, void* stream) {
  if (!d_W || !d_out) return set_error(MVB_ERR_ARG, "null argument");
  if (M < 1 || (fmt == WFmt::FP8 && M % 2) || K < 256 || K % 256) return set_error(MVB_ERR_ARG, "bad shape M=%d K=%d", M, K);
  WidenBatch m{};
  m.src[0] = reinterpret_cast<const uint8_t*>(d_W);
  m.dst[0] = reinterpret_cast<__nv_bfloat16*>(d_out);
  m.M[0] = M; m.K[0] = K; m.n = 1;
  int dev = 0, n_sm = 0;
  if (int e = current_device(&dev, &n_sm)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  MVB_CK(widen(fmt, m, n_sm, s));
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}

extern "C" int mvb_w4_dequant_test(const void* d_W, int32_t M, int32_t K, void* d_out, void* stream) {
  return widen_test(WFmt::INT4, d_W, M, K, d_out, stream);
}

extern "C" int mvb_w8_widen_test(const void* d_W, int32_t M, int32_t K, void* d_out, void* stream) {
  return widen_test(WFmt::INT8, d_W, M, K, d_out, stream);
}

extern "C" int mvb_f8_widen_test(const void* d_W, int32_t M, int32_t K, void* d_out, void* stream) {
  return widen_test(WFmt::FP8, d_W, M, K, d_out, stream);
}

// Test hook of the fp8 KV store (include/mvb200.h): k_kv_store_f8 as path B launches it, over R caller-described rows.
extern "C" int mvb_s1_kv_f8_store_test(const float* d_qkv, int32_t R, int32_t H, int32_t n_cache_rows, int32_t S_max,
                                       const int32_t* d_cache_row, const int32_t* d_pos, void* d_codes, void* d_scales,
                                       void* stream) {
  if (!d_qkv || !d_cache_row || !d_pos || !d_codes || !d_scales) return set_error(MVB_ERR_ARG, "null argument");
  if (R < 1 || R > RB_MAX || H < 1 || n_cache_rows < 1 || S_max < 1)
    return set_error(MVB_ERR_ARG, "mvb_s1_kv_f8_store_test: R %d (1..%d), H %d, n_cache_rows %d, S_max %d", R, RB_MAX, H,
                     n_cache_rows, S_max);
  const size_t n_vec = (size_t)n_cache_rows * H * S_max;
  uint8_t* codes = reinterpret_cast<uint8_t*>(d_codes);
  __nv_bfloat16* scales = reinterpret_cast<__nv_bfloat16*>(d_scales);
  const KvF8 kv{codes, codes + n_vec * 128, scales, scales + n_vec};
  RowsDev rw{};
  rw.cache_row = const_cast<int*>(d_cache_row);
  rw.pos = const_cast<int*>(d_pos);
  cudaStream_t s = (cudaStream_t)stream;
  k_kv_store_f8<true><<<(2 * R * H + 7) / 8, 256, 0, s>>>(S1State{}, rw, R, d_qkv, kv, H, S_max, 128 * H);
  MVB_CK(cudaGetLastError());
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}

// ------------------------------------------------------------------------------------------------
// Test hook of the non-production architectures' projections (include/mvb200.h): k_gemv with any norm, bias and epilogue
// exactly as path A launches it, or the BIASED QKV k_tc_gemm of path B with a forced K split.
// Rows of a tensor-core QKV test: activation row n -> cache row 2 s + (n & 1) at position pos[s], s = slot_map[n >> 1].
__global__ void k_rows_of_slots(const int* __restrict__ slot_map, const int* __restrict__ pos, int n_utts,
                                int* __restrict__ row_cache, int* __restrict__ row_pos) {
  const int n = threadIdx.x;
  if (n < 2 * n_utts) {
    const int s = slot_map[n >> 1];
    row_cache[n] = 2 * s + (n & 1);
    row_pos[n] = pos[s];
  }
}

extern "C" int mvb_s1_arch_gemv_test(int32_t path, int32_t epi, int32_t norm, const void* d_W, const void* d_W3,
                                     const void* d_bias, const void* d_bias3, int32_t M, int32_t K, const float* d_x,
                                     int32_t ldx, int32_t n_utts, const void* d_gain, const void* d_beta, float eps,
                                     float* d_out, int32_t ldo, void* d_kcache, void* d_vcache, const int32_t* d_slot_map,
                                     const int32_t* d_pos, int32_t H, int32_t S_max, int32_t D, int32_t kv_fp32,
                                     int32_t ksplit_override, void* stream) {
  if (!d_W || !d_x || !d_out || !d_slot_map || !d_pos) return set_error(MVB_ERR_ARG, "null argument");
  if (path != 0 && path != 1) return set_error(MVB_ERR_ARG, "mvb_s1_arch_gemv_test: path %d", path);
  if (epi < EPI_STORE || epi > EPI_GELU) return set_error(MVB_ERR_ARG, "mvb_s1_arch_gemv_test: epilogue %d", epi);
  if (norm < 0 || norm > 2) return set_error(MVB_ERR_ARG, "mvb_s1_arch_gemv_test: norm %d", norm);
  if ((norm != 0) != (d_gain != nullptr) || (d_beta && norm != 2))
    return set_error(MVB_ERR_ARG, "mvb_s1_arch_gemv_test: a norm takes a gain (and only LayerNorm a beta)");
  if (n_utts < 1 || n_utts > 64) return set_error(MVB_ERR_ARG, "mvb_s1_arch_gemv_test: n_utts %d", n_utts);
  if (epi == EPI_SWIGLU && (!d_W3 || (d_bias && !d_bias3)))
    return set_error(MVB_ERR_ARG, "mvb_s1_arch_gemv_test: SwiGLU needs W3 (and bias3 with a bias)");
  if (epi == EPI_QKV && (!d_kcache || !d_vcache || M != 3 * D || D != 128 * H || S_max < 1))
    return set_error(MVB_ERR_ARG, "mvb_s1_arch_gemv_test: QKV needs both caches, D == 128 H, M == 3 D, S_max >= 1");
  if (ldo < M || ldx < K) return set_error(MVB_ERR_ARG, "mvb_s1_arch_gemv_test: ldo >= M and ldx >= K required");
  cudaStream_t s = (cudaStream_t)stream;
  if (path == 1) {
    if (epi != EPI_QKV) return set_error(MVB_ERR_ARG, "mvb_s1_arch_gemv_test: path 1 is the QKV GEMM");
    if (K % 64 || 2 * n_utts > RB_MAX) return set_error(MVB_ERR_UNSUPPORTED, "mvb_s1_arch_gemv_test: K %% 64 == 0, 2 n_utts <= 128");
    int* rows = nullptr;
    MVB_CK(cudaMalloc(&rows, sizeof(int) * 2 * RB_MAX));
    k_rows_of_slots<<<1, RB_MAX, 0, s>>>(d_slot_map, d_pos, n_utts, rows, rows + RB_MAX);
    TcGemm a{};
    a.epi = G_QKV;
    a.x = d_x; a.ldx = ldx; a.gain = reinterpret_cast<const __nv_bfloat16*>(d_gain); a.eps = eps;
    a.layer_norm = norm == 2; a.beta = reinterpret_cast<const __nv_bfloat16*>(d_beta);
    a.M = M; a.K = K; a.R = 2 * n_utts; a.split_lo = 1; a.ksplit = ksplit_override;
    a.out = d_out; a.ldo = ldo;
    a.kcache = d_kcache; a.vcache = d_vcache; a.row_cache = rows; a.row_pos = rows + RB_MAX;
    a.H = H; a.S_max = S_max; a.D = D; a.kv_fp32 = kv_fp32;
    a.bias = reinterpret_cast<const __nv_bfloat16*>(d_bias);
    const cudaError_t le = cudaGetLastError();
    const int rc = le == cudaSuccess ? tc_gemm_test(a, d_W, nullptr, stream)
                                     : set_error(MVB_ERR_CUDA, "k_rows_of_slots: %s", cudaGetErrorString(le));
    cudaFree(rows);
    return rc;
  }
  if (K < 256 || K % 256 || M < 2 || M % 2 || (size_t)2 * K * sizeof(float) > GEMV_MAX_SMEM)
    return set_error(MVB_ERR_UNSUPPORTED, "mvb_s1_arch_gemv_test: bad GEMV shape M=%d K=%d", M, K);
  return gemv_test(WFmt::BF16, epi, norm == 2, d_W, d_W3, d_bias, d_bias3, M, K, d_x, ldx, n_utts, d_gain, d_beta, eps, d_out,
                   ldo, d_kcache, d_vcache, d_slot_map, d_pos, H, S_max, D, kv_fp32, s);
}
