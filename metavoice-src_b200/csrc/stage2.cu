// Stage 2: the non-causal codebook-expansion transformer (SURVEY.md rows a13-a15).
//   GPT.forward, causal=False      fam/llm/model.py:195-314   (sum of hierarchy embeddings + wpe + speaker)
//   Block / SelfAttention / MLP    fam/llm/layers/combined.py:40-52, attn.py:122-185, layers.py:36-72
//   _non_causal_sample             fam/llm/mixins/non_causal.py:15-67 (temperature, top-k, softmax, multinomial)
// Every Linear runs on the TMA + mma.sync weight-streaming GEMM (tc_gemm, linear.cu; 128 activation rows per pass,
// hi+lo bf16 activations); attention is a full bidirectional softmax over the block (no padding mask, as in
// the reference); sampling is one CTA per (hierarchy, position).
#include <cuda_runtime.h>

#include <vector>

#include "common.cuh"
#include "host.cuh"
#include "tc_gemm_host.cuh"

using namespace mvb;

namespace {

constexpr int S2_ROWS = 128;   // activation rows per tensor-core pass

// x[row] = sum_h wte_h[idx[b, h, i]] + wpe[i] + W_spk . spk[b]      (model.py:232-236, 258-283)
__global__ void __launch_bounds__(128) k_s2_embed(const int* __restrict__ idx, int n_in, int t, const __nv_bfloat16* const* wte,
                                                  const __nv_bfloat16* __restrict__ wpe, const float* __restrict__ spk_proj,
                                                  float* __restrict__ x, int E) {
  const int row = blockIdx.x, b = row / t, i = row - b * t;
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    float v = 0.f;
    for (int h = 0; h < n_in; ++h) v += bf16_to_f32(wte[h][(size_t)idx[((size_t)b * n_in + h) * t + i] * E + e]);
    v += bf16_to_f32(wpe[(size_t)i * E + e]);
    if (spk_proj) v += spk_proj[(size_t)b * E + e];
    x[(size_t)row * E + e] = v;
  }
}

__global__ void __launch_bounds__(256) k_s2_spk(const __nv_bfloat16* __restrict__ W, const float* __restrict__ spk, float* __restrict__ out,
                                                int E, int SD) {
  const int b = blockIdx.y;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= E) return;
  float acc = 0.f;
  for (int k = lane; k < SD; k += 32) acc = fmaf(bf16_to_f32(W[(size_t)warp * SD + k]), spk[(size_t)b * SD + k], acc);
  acc = warp_sum(acc);
  if (lane == 0) out[(size_t)b * E + warp] = acc;
}

// Bidirectional attention (attn.py:148-155 with is_causal=False).  A CTA owns 32 queries of one head; every query is
// carried by a group of 4 lanes (each lane keeps HS/4 dimensions of q and of the output, scores are completed with two
// shuffles), K/V tiles of 64 keys are staged in shared memory (64 / 32 keys per tile) with 128-bit loads and broadcast to the 8 queries of a warp.
template <int HS>
__global__ void __launch_bounds__(128) k_s2_attn(const float* __restrict__ qkv, float* __restrict__ out, int t, int E, int n_head) {
  constexpr int DL = HS / 4;            // dimensions per lane
  constexpr int KT = HS == 64 ? 64 : 32;   // keys per tile (32 KB of static shared memory either way)
  __shared__ __align__(16) float sk[KT][HS];
  __shared__ __align__(16) float sv[KT][HS];
  const int h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, part = tid & 3;
  const int qi = blockIdx.x * 32 + (tid >> 2);
  const bool active = qi < t;
  const float scale = rsqrtf((float)HS);
  float q[DL], o[DL];
  const float* qp = qkv + ((size_t)b * t + (active ? qi : 0)) * 3 * E + h * HS + part * DL;
#pragma unroll
  for (int d = 0; d < DL; d += 4) {
    const float4 v = *reinterpret_cast<const float4*>(qp + d);
    q[d] = v.x * scale; q[d + 1] = v.y * scale; q[d + 2] = v.z * scale; q[d + 3] = v.w * scale;
    o[d] = o[d + 1] = o[d + 2] = o[d + 3] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  for (int k0 = 0; k0 < t; k0 += KT) {
    __syncthreads();
    for (int i = tid; i < KT * HS / 4; i += 128) {
      const int kk = i / (HS / 4), d4 = i - kk * (HS / 4);
      const bool ok = k0 + kk < t;
      const float* kp = qkv + ((size_t)b * t + (ok ? k0 + kk : 0)) * 3 * E + E + h * HS + d4 * 4;
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      reinterpret_cast<float4*>(&sk[kk][0])[d4] = ok ? *reinterpret_cast<const float4*>(kp) : z;
      reinterpret_cast<float4*>(&sv[kk][0])[d4] = ok ? *reinterpret_cast<const float4*>(kp + E) : z;
    }
    __syncthreads();
    const int nk = min(KT, t - k0);
    for (int kk = 0; kk < nk; kk += 4) {           // 4 keys per trip: independent score chains
      float sc[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float a = 0.f;
        const float* kr = &sk[kk + j][part * DL];
#pragma unroll
        for (int d = 0; d < DL; ++d) a = fmaf(q[d], kr[d], a);
        sc[j] = a;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        sc[j] += __shfl_xor_sync(0xffffffffu, sc[j], 1);
        sc[j] += __shfl_xor_sync(0xffffffffu, sc[j], 2);
        if (kk + j >= nk) sc[j] = -INFINITY;
      }
      const float mx = fmaxf(fmaxf(m, fmaxf(sc[0], sc[1])), fmaxf(sc[2], sc[3]));
      const float corr = __expf(m - mx);
      float pw[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) pw[j] = __expf(sc[j] - mx);
      l = l * corr + (pw[0] + pw[1]) + (pw[2] + pw[3]);
#pragma unroll
      for (int d = 0; d < DL; ++d) {
        float acc = o[d] * corr;
#pragma unroll
        for (int j = 0; j < 4; ++j) acc = fmaf(pw[j], sv[kk + j][part * DL + d], acc);
        o[d] = acc;
      }
      m = mx;
    }
  }
  if (active) {
    float* op = out + ((size_t)b * t + qi) * E + h * HS + part * DL;
    const float inv = 1.f / l;
#pragma unroll
    for (int d = 0; d < DL; d += 4)
      *reinterpret_cast<float4*>(op + d) = make_float4(o[d] * inv, o[d + 1] * inv, o[d + 2] * inv, o[d + 3] * inv);
  }
}

// _non_causal_sample for one (hierarchy, row): logits / T, top-k threshold, softmax, argmax(p / Exp(1)).
constexpr int S2_PAD = 2048;
struct S2SampleParams {   // lives in device memory so that a captured graph can be replayed with new values
  float temperature;
  int top_k;
  unsigned long long seed;
};
__global__ void __launch_bounds__(256) k_s2_sample(const float* __restrict__ logits, int V, const S2SampleParams* __restrict__ prm,
                                                   const float* __restrict__ noise, int* __restrict__ out, int n_rows) {
  const float temperature = prm->temperature;
  const int top_k = prm->top_k;
  const unsigned long long seed = prm->seed;
  __shared__ float key[S2_PAD];
  __shared__ float red[8];
  __shared__ unsigned long long rbest[8];
  const int row = blockIdx.x, hier = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* lg = logits + ((size_t)hier * n_rows + row) * V;
  for (int v = tid; v < S2_PAD; v += 256) key[v] = v < V ? __fdiv_rn(lg[v], temperature) : -INFINITY;
  __syncthreads();
  float pivot = -INFINITY;
  if (top_k > 0 && top_k < V) {
    // descending bitonic sort of a copy is avoided: sort in place, logits are re-read afterwards
    for (int k = 2; k <= S2_PAD; k <<= 1)
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int tt = tid; tt < S2_PAD / 2; tt += 256) {
          const int i = ((tt & ~(j - 1)) << 1) | (tt & (j - 1));
          const int ixj = i | j;
          const bool desc = ((i & k) == 0);
          const float a = key[i], b = key[ixj];
          if ((a < b) == desc) { key[i] = b; key[ixj] = a; }
        }
        __syncthreads();
      }
    pivot = key[top_k - 1];   // k-th largest (non_causal.py:43-44: logits < v[..., -1] -> -inf)
    __syncthreads();
  }
  // softmax over kept logits
  float mx = -INFINITY;
  for (int v = tid; v < V; v += 256) {
    const float x = __fdiv_rn(lg[v], temperature);
    if (x >= pivot) mx = fmaxf(mx, x);
  }
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int v = tid; v < V; v += 256) {
    const float x = __fdiv_rn(lg[v], temperature);
    if (x >= pivot) sum += expf(x - mx);
  }
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) sum += red[i];
  unsigned long long best = 0ull;
  for (int v = tid; v < V; v += 256) {
    const float x = __fdiv_rn(lg[v], temperature);
    const float pr = x >= pivot ? expf(x - mx) / sum : 0.f;
    float qv;
    if (noise) {
      qv = noise[((size_t)hier * n_rows + row) * V + v];
    } else {
      const uint4 r = philox4x32_10(make_uint4((unsigned)v, (unsigned)row, (unsigned)hier, 0x5eed2u),
                                    make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
      qv = philox_exp1(r.x);
    }
    const unsigned long long cand =
        ((unsigned long long)__float_as_uint(__fdiv_rn(pr, qv)) << 32) | (unsigned long long)(0xffffffffu - (unsigned)v);
    best = cand > best ? cand : best;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long n = __shfl_xor_sync(0xffffffffu, best, o);
    best = n > best ? n : best;
  }
  if (lane == 0) rbest[warp] = best;
  __syncthreads();
  if (tid == 0) {
#pragma unroll
    for (int i = 1; i < 8; ++i) best = rbest[i] > best ? rbest[i] : best;
    out[(size_t)hier * n_rows + row] = (int)(0xffffffffu - (unsigned)(best & 0xffffffffull));
  }
}

}  // namespace

// Per-layer norm parameters and Linear biases (null when the architecture has none).
struct S2LayerP {
  const __nv_bfloat16 *g1, *b1, *g2, *b2;                // ln_1 / ln_2 gain and (LayerNorm with bias) beta
  const __nv_bfloat16 *qkv_b, *o_b, *fc_b, *fc3_b, *proj_b;   // c_attn, attn.c_proj, c_fc | w1, w3, mlp.c_proj
};

struct mvb_s2 {
  mvb_s2_config cfg;
  mvb_s2_arch arch{};
  int n_sm = 132, hidden = 0;
  const char* arena = nullptr;
  std::vector<uint64_t> off;
  char* ws = nullptr;
  // workspace slices
  float *x, *qkv, *att, *ffn, *logits, *spk_proj, *scratch;
  __nv_bfloat16* B;
  unsigned* tickets;
  int* tokens;
  int* idx_stage;          // [max_batch, n_in, t] inputs copied here so that the captured graph only touches internal buffers
  float* spk_stage;        // [max_batch, spk_dim]
  S2SampleParams* params;  // device copy of the sampling parameters
  S2SampleParams* h_params = nullptr;   // pinned
  bool use_graph = true;
  cudaStream_t cap_stream = nullptr;
  cudaGraphExec_t graphs[2][65] = {};   // [has speaker][batch]
  const __nv_bfloat16** wte_dev;
  std::vector<CUtensorMap> tmW;   // per layer {c_attn, c_proj, w1 | c_fc, w3 (GELU: c_fc again), mlp.c_proj}, then heads
  CUtensorMap tmB_E, tmB_H;
  std::vector<S2LayerP> lp;
  const __nv_bfloat16* lnf_b = nullptr;
  const __nv_bfloat16* w(int i) const { return reinterpret_cast<const __nv_bfloat16*>(arena + off[i]); }
  bool gelu() const { return arch.mlp == MVB_S2_MLP_GELU; }
  // arena order: wte[n_in], wpe, spk_proj, ln_f, heads[n_out], then per layer {ln_1, c_attn, c_proj, ln_2, w1, w3, c_proj}
  // (GELU: {ln_1, c_attn, c_proj, ln_2, c_fc, c_proj}), then the biases (s2_offset_count)
  int g_wpe() const { return cfg.n_in; }
  int g_spk() const { return cfg.n_in + 1; }
  int g_lnf() const { return cfg.n_in + 2; }
  int g_head(int i) const { return cfg.n_in + 3 + i; }
  int g_layer(int l, int t) const { return cfg.n_in + 3 + cfg.n_out + l * (gelu() ? 6 : 7) + t; }
};

// Tensors in the offset list: the weights, then, with bias, ln_f.bias (LayerNorm) and per layer {ln_1.bias (LayerNorm),
// c_attn.bias, attn.c_proj.bias, ln_2.bias (LayerNorm), w1.bias, w3.bias | c_fc.bias, mlp.c_proj.bias}.
static int s2_offset_count(const mvb_s2_config* c, const mvb_s2_arch& a) {
  const bool ln = a.norm == MVB_S2_NORM_LAYER, gelu = a.mlp == MVB_S2_MLP_GELU;
  int n = c->n_in + 3 + c->n_out + c->n_layer * (gelu ? 6 : 7);
  if (a.bias) n += (ln ? 1 : 0) + c->n_layer * ((ln ? 2 : 0) + 3 + (gelu ? 1 : 2));
  return n;
}

static int s2_validate_arch(const mvb_s2_arch& a) {
  if (a.norm != MVB_S2_NORM_RMS && a.norm != MVB_S2_NORM_LAYER) return mvb::set_error(MVB_ERR_ARG, "arch.norm: undefined value %d", a.norm);
  if (a.mlp != MVB_S2_MLP_SWIGLU && a.mlp != MVB_S2_MLP_GELU) return mvb::set_error(MVB_ERR_ARG, "arch.mlp: undefined value %d", a.mlp);
  if (a.bias != 0 && a.bias != 1) return mvb::set_error(MVB_ERR_ARG, "arch.bias: undefined value %d", a.bias);
  return MVB_OK;
}

struct S2Layout { size_t x, qkv, att, ffn, logits, spk, B, scratch, tickets, tokens, wte, idx, spk_stage, params, total; };

static S2Layout s2_layout(const mvb_s2_config* c) {
  const size_t rows = (size_t)c->max_batch * c->block_size, E = c->n_embd, Hd = c->hidden;
  size_t vmax = 0;
  for (int i = 0; i < c->n_out; ++i) vmax = vmax > (size_t)c->vocab_out[i] ? vmax : (size_t)c->vocab_out[i];
  S2Layout L;
  WsBump ws;
  L.x = ws.take(rows * E * 4);
  L.qkv = ws.take(rows * 3 * E * 4);
  L.att = ws.take(rows * E * 4);
  L.ffn = ws.take(rows * Hd * 4);
  L.logits = ws.take((size_t)c->n_out * rows * vmax * 4);
  L.spk = ws.take((size_t)c->max_batch * E * 4);
  L.B = ws.take((size_t)2 * S2_ROWS * (Hd > E ? Hd : E) * 2);
  size_t sc = 0;
  const size_t mats[5][3] = {{3 * E, E, 1}, {E, E, 1}, {Hd, E, 2}, {E, Hd, 1}, {vmax, E, 1}};
  for (auto& m : mats) {
    GemmPlan g = plan_gemm((int)m[0], (int)m[1], 2 * S2_ROWS, m[2] == 2, GEMM_MAX_SM);
    sc = sc > g.scratch_floats ? sc : g.scratch_floats;
  }
  L.scratch = ws.take(sc * 4);
  L.tickets = ws.take(256 * 4);
  L.tokens = ws.take((size_t)c->n_out * rows * 4);
  L.wte = ws.take(16 * sizeof(void*));
  L.idx = ws.take((size_t)c->max_batch * c->n_in * c->block_size * 4);
  L.spk_stage = ws.take((size_t)c->max_batch * c->spk_dim * 4);
  L.params = ws.take(256);
  L.total = ws.end;
  return L;
}

static int s2_validate(const mvb_s2_config* c) {
  if (!c) return mvb::set_error(MVB_ERR_ARG, "null config");
  if (c->n_embd % 64 || c->hidden % 64) return mvb::set_error(MVB_ERR_UNSUPPORTED, "n_embd and hidden must be multiples of 64");
  const int hs = c->n_embd / c->n_head;
  if (hs * c->n_head != c->n_embd || (hs != 64 && hs != 128)) return mvb::set_error(MVB_ERR_UNSUPPORTED, "head size must be 64 or 128");
  if (c->n_in < 1 || c->n_in > 8 || c->n_out < 1 || c->n_out > 8) return mvb::set_error(MVB_ERR_ARG, "hierarchy counts out of range");
  for (int i = 0; i < c->n_out; ++i)
    if (c->vocab_out[i] > S2_PAD) return mvb::set_error(MVB_ERR_UNSUPPORTED, "target vocab > %d", S2_PAD);
  if (c->max_batch < 1 || c->max_batch > 64 || c->block_size < 1) return mvb::set_error(MVB_ERR_ARG, "bad batch / block size");
  if (c->options & ~MVB_S2_EAGER)
    return mvb::set_error(MVB_ERR_ARG, "options: undefined bits 0x%x", (unsigned)(c->options & ~MVB_S2_EAGER));
  return MVB_OK;
}

extern "C" size_t mvb_s2_workspace_bytes(const mvb_s2_config* c) {
  if (s2_validate(c)) return 0;
  return s2_layout(c).total;
}

extern "C" int mvb_s2_create_ex(const mvb_s2_config* cfg, const mvb_s2_arch* arch, const void* d_arena, size_t arena_bytes,
                                const uint64_t* offsets, void* d_ws, mvb_s2** out) {
  if (int e = s2_validate(cfg)) return e;
  const mvb_s2_arch a = arch ? *arch : mvb_s2_arch{};
  if (int e = s2_validate_arch(a)) return e;
  if (!offsets) return mvb::set_error(MVB_ERR_ARG, "null pointer argument");
  const int n_off = s2_offset_count(cfg, a);
  if (int e = check_offsets(offsets, n_off, arena_bytes, "stage 2: weight offset")) return e;
  if (!d_arena || !d_ws || !out) return mvb::set_error(MVB_ERR_ARG, "null pointer argument");
  Building<mvb_s2> hb(new mvb_s2(), mvb_s2_destroy);
  mvb_s2* h = hb.get();
  h->cfg = *cfg;
  h->arch = a;
  h->hidden = cfg->hidden;
  int dev = 0;
  if (int e = current_device(&dev, &h->n_sm)) return e;
  h->arena = reinterpret_cast<const char*>(d_arena);
  h->off.assign(offsets, offsets + n_off);
  h->ws = reinterpret_cast<char*>(d_ws);
  const S2Layout L = s2_layout(cfg);
  h->idx_stage = (int*)(h->ws + L.idx); h->spk_stage = (float*)(h->ws + L.spk_stage); h->params = (S2SampleParams*)(h->ws + L.params);
  h->use_graph = !(cfg->options & MVB_S2_EAGER);
  h->x = (float*)(h->ws + L.x); h->qkv = (float*)(h->ws + L.qkv); h->att = (float*)(h->ws + L.att); h->ffn = (float*)(h->ws + L.ffn);
  h->logits = (float*)(h->ws + L.logits); h->spk_proj = (float*)(h->ws + L.spk); h->B = (__nv_bfloat16*)(h->ws + L.B);
  h->scratch = (float*)(h->ws + L.scratch); h->tickets = (unsigned*)(h->ws + L.tickets); h->tokens = (int*)(h->ws + L.tokens);
  h->wte_dev = (const __nv_bfloat16**)(h->ws + L.wte);
  std::vector<const __nv_bfloat16*> wte(cfg->n_in);
  for (int i = 0; i < cfg->n_in; ++i) wte[i] = h->w(i);
  MVB_CK(cudaMemcpy(h->wte_dev, wte.data(), sizeof(void*) * cfg->n_in, cudaMemcpyHostToDevice));
  const int E = cfg->n_embd, Hd = h->hidden;
  const bool ln = a.norm == MVB_S2_NORM_LAYER, gelu = h->gelu();
  int nb = s2_offset_count(cfg, mvb_s2_arch{a.norm, a.mlp, 0});    // first bias slot
  auto bias_slot = [&](bool present) { return present && a.bias ? h->w(nb++) : nullptr; };
  h->lnf_b = bias_slot(ln);
  h->lp.resize(cfg->n_layer);
  for (int l = 0; l < cfg->n_layer; ++l) {
    S2LayerP& p = h->lp[l];
    p.g1 = h->w(h->g_layer(l, 0));
    p.g2 = h->w(h->g_layer(l, 3));
    p.b1 = bias_slot(ln);
    p.qkv_b = bias_slot(true);
    p.o_b = bias_slot(true);
    p.b2 = bias_slot(ln);
    p.fc_b = bias_slot(true);
    p.fc3_b = bias_slot(!gelu);
    p.proj_b = bias_slot(true);
  }
  h->tmW.resize((size_t)cfg->n_layer * 5 + cfg->n_out);
  bool ok = true;
  for (int l = 0; l < cfg->n_layer && ok; ++l) {
    ok = ok && make_tmap_bf16(&h->tmW[l * 5 + 0], h->w(h->g_layer(l, 1)), 3 * E, E, 128);
    ok = ok && make_tmap_bf16(&h->tmW[l * 5 + 1], h->w(h->g_layer(l, 2)), E, E, 128);
    ok = ok && make_tmap_bf16(&h->tmW[l * 5 + 2], h->w(h->g_layer(l, 4)), Hd, E, 128);
    ok = ok && make_tmap_bf16(&h->tmW[l * 5 + 3], h->w(h->g_layer(l, gelu ? 4 : 5)), Hd, E, 128);
    ok = ok && make_tmap_bf16(&h->tmW[l * 5 + 4], h->w(h->g_layer(l, gelu ? 5 : 6)), E, Hd, 128);
  }
  for (int i = 0; i < cfg->n_out && ok; ++i)
    ok = ok && make_tmap_bf16(&h->tmW[(size_t)cfg->n_layer * 5 + i], h->w(h->g_head(i)), cfg->vocab_out[i], E, 128);
  ok = ok && make_tmap_bf16(&h->tmB_E, h->B, 2 * S2_ROWS, E, 2 * S2_ROWS);
  ok = ok && make_tmap_bf16(&h->tmB_H, h->B, 2 * S2_ROWS, Hd, 2 * S2_ROWS);
  if (!ok) return mvb::set_error(MVB_ERR_CUDA, "cuTensorMapEncodeTiled failed (stage 2)");
  if (cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMallocHost(&h->h_params, sizeof(S2SampleParams)) != cudaSuccess)
    return mvb::set_error(MVB_ERR_CUDA, "stage 2: stream / pinned buffer allocation failed");
  *out = hb.release();
  return MVB_OK;
}

extern "C" int mvb_s2_create(const mvb_s2_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets, void* d_ws,
                             mvb_s2** out) {
  return mvb_s2_create_ex(cfg, nullptr, d_arena, arena_bytes, offsets, d_ws, out);
}

extern "C" int mvb_s2_destroy(mvb_s2* h) {
  if (!h) return MVB_OK;
  for (auto& row : h->graphs)
    for (auto& g : row)
      if (g) cudaGraphExecDestroy(g);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  if (h->h_params) cudaFreeHost(h->h_params);
  delete h;
  return MVB_OK;
}

// Launches the front end exactly as s2_body does: the speaker projection spk_proj[b] = W_spk . spk[b] (when spk is
// non-null), then x[b*t + i] = sum_h wte_h[idx[b, h, i]] + wpe[i] (+ spk_proj[b]).
static cudaError_t launch_s2_embed(cudaStream_t s, const int* idx, int B, int n_in, int t, const __nv_bfloat16* const* wte,
                                   const __nv_bfloat16* wpe, const __nv_bfloat16* W_spk, const float* spk, int SD, int E,
                                   float* spk_proj, float* x) {
  if (spk) {
    k_s2_spk<<<dim3((E * 32 + 255) / 256, B), 256, 0, s>>>(W_spk, spk, spk_proj, E, SD);
    if (cudaError_t e = cudaGetLastError()) return e;
  }
  k_s2_embed<<<B * t, 128, 0, s>>>(idx, n_in, t, wte, wpe, spk ? spk_proj : nullptr, x, E);
  return cudaGetLastError();
}

extern "C" int mvb_s2_embed_test(const int32_t* d_idx, int32_t B, int32_t n_in, int32_t t, const void* d_wte, const void* d_wpe,
                                 const void* d_W_spk, const float* d_spk, int32_t spk_dim, int32_t E, float* d_spk_proj, float* d_x,
                                 void* stream) {
  if (!d_idx || !d_wte || !d_wpe || !d_x || (d_spk && (!d_W_spk || !d_spk_proj)))
    return mvb::set_error(MVB_ERR_ARG, "mvb_s2_embed_test: null argument");
  if (B < 1 || t < 1 || E < 1 || spk_dim < 1 || n_in < 1 || n_in > 8)
    return mvb::set_error(MVB_ERR_ARG, "mvb_s2_embed_test: B, t, E, spk_dim >= 1 and 1 <= n_in <= 8 required");
  cudaStream_t s = (cudaStream_t)stream;
  MVB_CK(launch_s2_embed(s, d_idx, B, n_in, t, reinterpret_cast<const __nv_bfloat16* const*>(d_wte),
                         reinterpret_cast<const __nv_bfloat16*>(d_wpe), reinterpret_cast<const __nv_bfloat16*>(d_W_spk), d_spk,
                         spk_dim, E, d_spk_proj, d_x));
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}

// Launches the bidirectional attention of one layer exactly as s2_body does.
static cudaError_t launch_s2_attn(cudaStream_t s, const float* qkv, float* out, int batch, int t, int E, int n_head) {
  const dim3 ag((t + 31) / 32, n_head, batch);
  if (E / n_head == 64) k_s2_attn<64><<<ag, 128, 0, s>>>(qkv, out, t, E, n_head);
  else k_s2_attn<128><<<ag, 128, 0, s>>>(qkv, out, t, E, n_head);
  return cudaGetLastError();
}

extern "C" int mvb_s2_attn_test(const float* d_qkv, int32_t B, int32_t t, int32_t E, int32_t n_head, float* d_out, void* stream) {
  if (!d_qkv || !d_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (B < 1 || t < 1 || n_head < 1 || E != n_head * (E / n_head) || (E / n_head != 64 && E / n_head != 128))
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_s2_attn_test: B, t >= 1 and head size E / n_head of 64 or 128 required");
  cudaStream_t s = (cudaStream_t)stream;
  MVB_CK(launch_s2_attn(s, d_qkv, d_out, B, t, E, n_head));
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}

// Launches the sampler over n_out hierarchies x rows logits rows of V entries exactly as s2_body does.
static cudaError_t launch_s2_sample(cudaStream_t s, const float* logits, int V, const S2SampleParams* prm, const float* noise,
                                    int* tokens, int rows, int n_out) {
  k_s2_sample<<<dim3(rows, n_out), 256, 0, s>>>(logits, V, prm, noise, tokens, rows);
  return cudaGetLastError();
}

extern "C" int mvb_s2_sample_test(const float* d_logits, int32_t n_hier, int32_t n_rows, int32_t V, const void* d_params,
                                  const float* d_noise, int32_t* d_tokens, void* stream) {
  if (!d_logits || !d_params || !d_tokens) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (n_hier < 1 || n_rows < 1 || V < 1 || V > S2_PAD)
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_s2_sample_test: n_hier, n_rows >= 1 and 1 <= V <= %d required", S2_PAD);
  cudaStream_t s = (cudaStream_t)stream;
  MVB_CK(launch_s2_sample(s, d_logits, V, reinterpret_cast<const S2SampleParams*>(d_params), d_noise, d_tokens, n_rows, n_hier));
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}

// y[rows, M] (+)= f(x)[rows, K] . W^T (+ bias) in passes of 128 rows through the tensor-core GEMM; f = the arch's norm
// (gain, beta) when gain != null.  LayerNorm's eps is 1e-5 (layers/layers.py:17), RMSNorm's the config's.
template <int EPI>
static int s2_linear(mvb_s2* h, cudaStream_t s, int rows, const float* x, int ldx, const __nv_bfloat16* gain,
                     const __nv_bfloat16* beta, int widx, int widx3, const __nv_bfloat16* bias, const __nv_bfloat16* bias3, int M,
                     int K, float* out, int ldo) {
  TcGemm g{};
  g.epi = EPI; g.Rpad = S2_ROWS; g.split_lo = 1;
  g.tmW = &h->tmW[widx]; g.tmW3 = &h->tmW[widx3];
  g.B = h->B; g.tmB = (K == h->cfg.n_embd) ? &h->tmB_E : &h->tmB_H;
  g.ldx = ldx; g.gain = gain;
  g.layer_norm = gain != nullptr && h->arch.norm == MVB_S2_NORM_LAYER;
  g.beta = g.layer_norm ? beta : nullptr;
  g.eps = g.layer_norm ? 1e-5f : h->cfg.norm_eps;
  g.bias = bias; g.bias3 = bias3;
  g.M = M; g.K = K; g.ldo = ldo;
  g.scratch = h->scratch; g.tickets = h->tickets; g.n_sm = h->n_sm;
  for (int r0 = 0; r0 < rows; r0 += S2_ROWS) {
    g.R = rows - r0 < S2_ROWS ? rows - r0 : S2_ROWS;
    g.x = x + (size_t)r0 * ldx;
    g.out = out + (size_t)r0 * ldo;
    MVB_CK(tc_gemm(s, g));
  }
  return MVB_OK;
}

// embed -> n_layer x {attention, MLP} -> ln_f + heads -> sampler, on internal buffers only (graph-capturable)
static int s2_body(mvb_s2* h, cudaStream_t s, int batch, bool has_spk, const float* d_noise) {
  const mvb_s2_config& c = h->cfg;
  const int t = c.block_size, rows = batch * t, E = c.n_embd, Hd = h->hidden;
  MVB_CK(cudaMemsetAsync(h->tickets, 0, 256 * 4, s));
  MVB_CK(launch_s2_embed(s, h->idx_stage, batch, c.n_in, t, h->wte_dev, h->w(h->g_wpe()), h->w(h->g_spk()),
                         has_spk ? h->spk_stage : nullptr, c.spk_dim, E, h->spk_proj, h->x));
  for (int l = 0; l < c.n_layer; ++l) {
    const S2LayerP& p = h->lp[l];
    if (int e = s2_linear<G_STORE>(h, s, rows, h->x, E, p.g1, p.b1, l * 5 + 0, l * 5 + 0, p.qkv_b, nullptr, 3 * E, E, h->qkv, 3 * E)) return e;
    MVB_CK(launch_s2_attn(s, h->qkv, h->att, batch, t, E, c.n_head));
    if (int e = s2_linear<G_RESID>(h, s, rows, h->att, E, nullptr, nullptr, l * 5 + 1, l * 5 + 1, p.o_b, nullptr, E, E, h->x, E)) return e;
    if (h->gelu()) {
      if (int e = s2_linear<G_GELU>(h, s, rows, h->x, E, p.g2, p.b2, l * 5 + 2, l * 5 + 2, p.fc_b, nullptr, Hd, E, h->ffn, Hd)) return e;
    } else {
      if (int e = s2_linear<G_SWIGLU>(h, s, rows, h->x, E, p.g2, p.b2, l * 5 + 2, l * 5 + 3, p.fc_b, p.fc3_b, Hd, E, h->ffn, Hd)) return e;
    }
    if (int e = s2_linear<G_RESID>(h, s, rows, h->ffn, Hd, nullptr, nullptr, l * 5 + 4, l * 5 + 4, p.proj_b, nullptr, E, Hd, h->x, E)) return e;
  }
  const int vmax = c.vocab_out[0];
  for (int i = 0; i < c.n_out; ++i) {
    const int hw = c.n_layer * 5 + i;
    if (int e = s2_linear<G_STORE>(h, s, rows, h->x, E, h->w(h->g_lnf()), h->lnf_b, hw, hw, nullptr, nullptr, vmax, E,
                                   h->logits + (size_t)i * rows * vmax, vmax)) return e;
  }
  MVB_CK(launch_s2_sample(s, h->logits, vmax, h->params, d_noise, h->tokens, rows, c.n_out));
  return MVB_OK;
}

extern "C" int mvb_s2_forward(mvb_s2* h, int32_t batch, const int32_t* d_idx, const float* d_spk, float temperature, int32_t top_k,
                              const float* d_noise, uint64_t seed, int32_t* d_tokens, float* d_logits_out, void* stream) {
  if (!h || !d_idx || !d_tokens) return mvb::set_error(MVB_ERR_ARG, "null argument");
  const mvb_s2_config& c = h->cfg;
  if (batch < 1 || batch > c.max_batch) return mvb::set_error(MVB_ERR_ARG, "batch %d out of range", batch);
  if (!(temperature > 0.f)) return mvb::set_error(MVB_ERR_ARG, "temperature must be positive");
  for (int i = 1; i < c.n_out; ++i)
    if (c.vocab_out[i] != c.vocab_out[0]) return mvb::set_error(MVB_ERR_UNSUPPORTED, "target vocabularies must be equal");
  cudaStream_t s = (cudaStream_t)stream;
  const int t = c.block_size, rows = batch * t;
  const size_t vmax = c.vocab_out[0];
  // inputs -> internal staging buffers: the forward pass itself (~500 small launches: 8 passes of 128 rows per Linear)
  // only touches library memory and is replayed as ONE CUDA graph per (batch, speaker) signature
  MVB_CK(cudaMemcpyAsync(h->idx_stage, d_idx, sizeof(int) * (size_t)batch * c.n_in * t, cudaMemcpyDeviceToDevice, s));
  if (d_spk) MVB_CK(cudaMemcpyAsync(h->spk_stage, d_spk, sizeof(float) * (size_t)batch * c.spk_dim, cudaMemcpyDeviceToDevice, s));
  MVB_CK(cudaStreamSynchronize(s));            // h_params is reused across calls: the previous upload must have been consumed
  h->h_params->temperature = temperature; h->h_params->top_k = top_k; h->h_params->seed = seed;
  MVB_CK(cudaMemcpyAsync(h->params, h->h_params, sizeof(S2SampleParams), cudaMemcpyHostToDevice, s));
  if (h->use_graph && d_noise == nullptr) {
    cudaGraphExec_t& ge = h->graphs[d_spk ? 1 : 0][batch];
    if (!ge) {
      auto body = [&](cudaStream_t cs) { return s2_body(h, cs, batch, d_spk != nullptr, nullptr); };
      if (int e = capture_graph(h->cap_stream, &ge, body)) return e;
    }
    MVB_CK(cudaGraphLaunch(ge, s));
  } else {
    if (int e = s2_body(h, s, batch, d_spk != nullptr, d_noise)) return e;
  }
  // tokens [n_out, batch*t] -> caller layout [batch, n_out, t]
  for (int b = 0; b < batch; ++b)
    for (int i = 0; i < c.n_out; ++i)
      MVB_CK(cudaMemcpyAsync(d_tokens + ((size_t)b * c.n_out + i) * t, h->tokens + (size_t)i * rows + (size_t)b * t, sizeof(int) * t,
                          cudaMemcpyDeviceToDevice, s));
  if (d_logits_out) MVB_CK(cudaMemcpyAsync(d_logits_out, h->logits, sizeof(float) * c.n_out * rows * vmax, cudaMemcpyDeviceToDevice, s));
  return MVB_OK;
}
