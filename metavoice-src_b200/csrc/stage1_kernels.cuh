// Stage-1 decode-path kernels, CUDA-core generation ("path A"): one kernel per operator, fp32
// activations, bf16 weights streamed once with 128-bit loads.  Each kernel cites the reference
// operator it replaces (metavoiceio/metavoice-src @ de3fa211).
//
// Row convention: utterance slot u owns activation rows 2u (speaker-conditioned) and 2u+1
// (unconditioned) -- the CFG pair of fam/llm/fast_model.py:132-134.
#pragma once
#include <type_traits>

#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "common.cuh"

namespace mvb {

// ---------------------------------------------------------------------------------------------
// Device-resident decode state (lives in the caller's workspace).  Everything the step needs is
// read from here so one captured CUDA graph can be replayed for every token.
struct SamplingDev {
  float guidance, temperature, top_p;
  int top_k, end_of_audio;
  // Prompt-guidance link (mvb_s1_admit_guided), in what would otherwise be padding: 0 = none, c + 1 on a guided primary
  // whose companion slot is c, -(u + 1) on the companion of primary u.  A companion's entry is not otherwise used for
  // sampling, so it carries the primary's prompt guidance scale p in `guidance` and end_of_text in `end_of_audio`.
  int link;
  unsigned long long seed;
};
static_assert(sizeof(SamplingDev) == 32, "SamplingDev is part of the pinned workspace layout");

struct S1State {
  int* slot_map;        // [max_utts] logical batch index -> utterance slot
  int* pos;             // [max_utts] cache position the current token is written to
  int* row_tok;         // [2*max_utts] token fed to each row this step
  int* done;            // [max_utts] end-of-audio latch (fast_inference_utils.py:161)
  int* n_gen;           // [max_utts] tokens produced so far
  int* gen_tokens;      // [max_utts, max_new] tokens fed back (== generate()'s appended tokens)
  int* sampled_tokens;  // [max_utts, max_new] tokens the sampler drew (differs only under teacher forcing)
  SamplingDev* samp;    // [max_utts]
  const float** noise;  // [max_utts] optional Exp(1) draws [max_new, vocab]
  const int** forced;   // [max_utts] optional teacher-forced tokens [max_new]
  unsigned* attn_ticket;  // [2*max_utts*n_head] split-KV arrival counters
  int* budget;          // [max_utts] tokens this utterance may produce (generate(): min(T + max_new, block) - T, utils:196-204)
  int* noise_base;      // [max_utts] generation step that row 0 of noise[u] belongs to (host-staged noise arrives in chunks)
  int max_new, block_size;
};

// ---------------------------------------------------------------------------------------------
// spk_proj[u] = W_spk . spk_emb   (fast_model.py:155 speaker_cond_pos, hoisted out of the step).  TW = __nv_bfloat16, or
// int8_t for an int8 engine.  bf16 row scales (`scale`: an int8 engine's, or an fp8 engine's over its widened q) multiply
// each output once after the sum; a bf16 engine passes none.
__device__ __forceinline__ float w_to_f32(__nv_bfloat16 w) { return bf16_to_f32(w); }
__device__ __forceinline__ float w_to_f32(int8_t w) { return (float)w; }

template <typename TW>
__global__ void __launch_bounds__(256) k_spk_proj(const TW* __restrict__ W, const float* __restrict__ spk,
                                                  float* __restrict__ out, int D, int SD, const __nv_bfloat16* __restrict__ scale) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= D) return;
  float acc = 0.f;
  for (int k = lane; k < SD; k += 32) acc = fmaf(w_to_f32(W[(size_t)warp * SD + k]), spk[k], acc);
  acc = warp_sum(acc);
  if (scale != nullptr) acc *= bf16_to_f32(scale[warp]);
  if (lane == 0) out[warp] = acc;
}

// Install the inputs of one forward position: == the (idx[:, s], input_pos[s]) arguments of
// Transformer.forward (fast_model.py:150).
__global__ void k_set_input(S1State st, int utt, const int* __restrict__ idx, int S, int s, int pos) {
  if (threadIdx.x == 0) {
    st.slot_map[0] = utt;
    st.pos[utt] = pos;
    st.row_tok[2 * utt] = idx[s];
    st.row_tok[2 * utt + 1] = idx[S + s];
  }
}

__global__ void k_begin(S1State st, int utt, int first_token, int pos, SamplingDev sp, const float* noise,
                        const int* forced, int has_first, int budget) {
  if (threadIdx.x == 0) {
    st.samp[utt] = sp;
    st.noise[utt] = noise;
    st.noise_base[utt] = 0;
    st.forced[utt] = forced;
    st.done[utt] = 0;
    st.n_gen[utt] = 0;
    st.pos[utt] = pos;
    st.budget[utt] = budget;
    if (has_first) {
      st.row_tok[2 * utt] = first_token;
      st.row_tok[2 * utt + 1] = first_token;
    }
  }
}

__global__ void k_identity_slots(S1State st, int n) {
  if ((int)threadIdx.x < n) st.slot_map[threadIdx.x] = threadIdx.x;
}

// ---------------------------------------------------------------------------------------------
// x = tok_emb[idx] + pos_emb[input_pos] + speaker_cond * mask      (fast_model.py:152-157)
// The reference has no RoPE: positions are a learned table (SURVEY.md D1).
__global__ void __launch_bounds__(256) k_embed(S1State st, const __nv_bfloat16* __restrict__ tok_emb,
                                               const __nv_bfloat16* __restrict__ pos_emb,
                                               const float* __restrict__ spk_proj, float* __restrict__ x, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int u = st.slot_map[blockIdx.y];
  const int c = blockIdx.x;  // 0 = conditioned row, 1 = unconditioned row
  const int r = 2 * u + c;
  const int tok = st.row_tok[r];
  const int pos = st.pos[u];
  const __nv_bfloat16* te = tok_emb + (size_t)tok * D;
  const __nv_bfloat16* pe = pos_emb + (size_t)pos * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float v = bf16_to_f32(te[d]) + bf16_to_f32(pe[d]);
    if (c == 0) v += spk_proj[(size_t)u * D + d];
    x[(size_t)r * D + d] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// Weight-streaming GEMV for the 2 CFG rows of one utterance, with the RMSNorm of
// fast_model.py:250-261 fused into the prologue and the operator-specific epilogue fused in:
//   EPI_QKV    : Attention.wqkv + KVCache.update scatter      (fast_model.py:206-215, 104-113)
//   EPI_RESID  : wo / w2 projection + residual add             (fast_model.py:226,179-180, 247)
//   EPI_SWIGLU : silu(w1 x) * (w3 x)                           (fast_model.py:230-237)
//   EPI_STORE  : final norm + LM head                          (fast_model.py:161-163)
//   EPI_GELU   : GELU(c_fc x), exact erf                       (layers/layers.py:45-48, 63-65: nn.GELU())
// The other GPTConfig architectures (model.py:26-46) add a LayerNorm prologue (k_gemv's LAYER flag) and the Linear
// biases of c_attn, attn.c_proj and the MLP (BIASED; attn.py:61-64, layers.py:37-53); the int4 / int8 GEMVs never take
// either.
enum { EPI_STORE = 0, EPI_RESID = 1, EPI_SWIGLU = 2, EPI_QKV = 3, EPI_GELU = 4 };

struct GemvP {
  const __nv_bfloat16* W;
  const __nv_bfloat16* W3;
  const float* x;
  int ldx;
  const __nv_bfloat16* gain;
  float eps;
  float* out;
  int ldo;
  int M, K;
  // EPI_QKV only
  void* kcache;
  void* vcache;
  int H, S_max, D, kv_fp32;
  // k_gemv only: LayerNorm beta [K] or null (LAYER), Linear biases of W (and W3) [M] (BIASED)
  const __nv_bfloat16* beta;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* bias3;
};

// nn.GELU(approximate='none'), as k_tc_gemm's G_GELU epilogue computes it
__device__ __forceinline__ float gelu_erf(float y) { return 0.5f * y * (1.f + erff(y * (float)M_SQRT1_2)); }

// Position of activation k inside the conflict-free shared-memory layout: a lane's eight
// consecutive k values are split into two float4 that sit 128 floats apart.
__device__ __forceinline__ int xs_perm(int k) {
  const int w = k & 255;
  return (k & ~255) + (((w & 7) >> 2) << 7) + ((w >> 3) << 2) + (w & 3);
}

template <int EPI>
__device__ __forceinline__ void gemv_rows(const GemvP& p, int item, int lane, const uint4*& wa, const uint4*& wb) {
  if (EPI == EPI_SWIGLU) {
    wa = reinterpret_cast<const uint4*>(p.W + (size_t)item * p.K) + lane;
    wb = reinterpret_cast<const uint4*>(p.W3 + (size_t)item * p.K) + lane;
  } else {
    wa = reinterpret_cast<const uint4*>(p.W + (size_t)(2 * item) * p.K) + lane;
    wb = wa + (p.K >> 3);
  }
}

// Prologue of the GEMV kernels (k_gemv, k_gemv_w4, k_gemv_w8): stage the two activation rows r0, r0 + 1 of p.x into
// xs [2][K] at perm(k), RMS-normalised (fp32 statistics, then the bf16 gain) when p.gain is set.  Ends with __syncthreads.
// LAYER (k_gemv only): LayerNorm instead (layers/layers.py:8-17, F.layer_norm with eps p.eps), the arithmetic of
// k_prep_b<true>: fp32 mean, then the biased variance as a second pass over the centred row, then
// ((x - mean) * rsqrt(var + eps)) * gain (+ beta when p.beta is set); p.gain is required.
template <bool LAYER = false, typename Perm>
__device__ __forceinline__ void gemv_prologue(const GemvP& p, int r0, float* xs, float* red, Perm perm) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = p.K;
  const float* x0 = p.x + (size_t)r0 * p.ldx;
  const float* x1 = x0 + p.ldx;
  if constexpr (LAYER) {
    float s0 = 0.f, s1 = 0.f;
    for (int k = tid; k < K; k += 256) {
      const float a = x0[k], b = x1[k];
      s0 += a;
      s1 += b;
      const int pk = perm(k);
      xs[pk] = a;
      xs[K + pk] = b;
    }
    s0 = warp_sum(s0);
    s1 = warp_sum(s1);
    if (lane == 0) {
      red[warp] = s0;
      red[8 + warp] = s1;
    }
    __syncthreads();
    float t0 = 0.f, t1 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      t0 += red[i];
      t1 += red[8 + i];
    }
    const float m0 = t0 / (float)K, m1 = t1 / (float)K;
    __syncthreads();                       // every thread has read red before it is reused
    float q0 = 0.f, q1 = 0.f;
    for (int k = tid; k < K; k += 256) {   // this thread's own staged entries
      const int pk = perm(k);
      const float d0 = xs[pk] - m0, d1 = xs[K + pk] - m1;
      q0 = fmaf(d0, d0, q0);
      q1 = fmaf(d1, d1, q1);
    }
    q0 = warp_sum(q0);
    q1 = warp_sum(q1);
    if (lane == 0) {
      red[warp] = q0;
      red[8 + warp] = q1;
    }
    __syncthreads();
    t0 = 0.f;
    t1 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      t0 += red[i];
      t1 += red[8 + i];
    }
    const float rs0 = rsqrtf(t0 / (float)K + p.eps);
    const float rs1 = rsqrtf(t1 / (float)K + p.eps);
    for (int k = tid; k < K; k += 256) {
      const float g = bf16_to_f32(p.gain[k]);
      const int pk = perm(k);
      float v0 = ((xs[pk] - m0) * rs0) * g, v1 = ((xs[K + pk] - m1) * rs1) * g;
      if (p.beta != nullptr) {
        const float be = bf16_to_f32(p.beta[k]);
        v0 += be;
        v1 += be;
      }
      xs[pk] = v0;
      xs[K + pk] = v1;
    }
    __syncthreads();
    return;
  }
  float s0 = 0.f, s1 = 0.f;
  for (int k = tid; k < K; k += 256) {
    const float a = x0[k], b = x1[k];
    s0 = fmaf(a, a, s0);
    s1 = fmaf(b, b, s1);
    const int pk = perm(k);
    xs[pk] = a;
    xs[K + pk] = b;
  }
  if (p.gain != nullptr) {
    s0 = warp_sum(s0);
    s1 = warp_sum(s1);
    if (lane == 0) {
      red[warp] = s0;
      red[8 + warp] = s1;
    }
    __syncthreads();
    float t0 = 0.f, t1 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      t0 += red[i];
      t1 += red[8 + i];
    }
    const float rs0 = rsqrtf(t0 / (float)K + p.eps);
    const float rs1 = rsqrtf(t1 / (float)K + p.eps);
    for (int k = tid; k < K; k += 256) {
      const float g = bf16_to_f32(p.gain[k]);
      const int pk = perm(k);
      xs[pk] = (xs[pk] * rs0) * g;
      xs[K + pk] = (xs[K + pk] * rs1) * g;
    }
  }
  __syncthreads();
}

// Epilogue of the GEMV kernels for one item of slot u: a<weight row><activation row>, weight rows 2 item, 2 item + 1
// (EPI_SWIGLU: a0* = w1 row item, a1* = w3 row item).  BIASED (k_gemv only): the Linear biases are added to the sums
// first, so the QKV scatter stores k and v with their bias (before a bf16 cache rounds them).
template <int EPI, bool BIASED = false>
__device__ __forceinline__ void gemv_epilogue(const GemvP& p, const S1State& st, int u, int item, float a00, float a01,
                                              float a10, float a11) {
  const int r0 = 2 * u;
  float* o0 = p.out + (size_t)r0 * p.ldo;
  float* o1 = o0 + p.ldo;
  if constexpr (BIASED) {
    const float b0 = bf16_to_f32(p.bias[EPI == EPI_SWIGLU ? item : 2 * item]);
    const float b1 = bf16_to_f32(EPI == EPI_SWIGLU ? p.bias3[item] : p.bias[2 * item + 1]);
    a00 += b0;
    a01 += b0;
    a10 += b1;
    a11 += b1;
  }
  if (EPI == EPI_SWIGLU) {
    o0[item] = (a00 / (1.f + expf(-a00))) * a10;
    o1[item] = (a01 / (1.f + expf(-a01))) * a11;
  } else if (EPI == EPI_GELU) {
    const int j = 2 * item;
    o0[j] = gelu_erf(a00);
    o1[j] = gelu_erf(a01);
    o0[j + 1] = gelu_erf(a10);
    o1[j + 1] = gelu_erf(a11);
  } else {
    const int j = 2 * item;
    if (EPI == EPI_RESID) {
      o0[j] += a00;
      o1[j] += a01;
      o0[j + 1] += a10;
      o1[j + 1] += a11;
    } else {
      o0[j] = a00;
      o1[j] = a01;
      o0[j + 1] = a10;
      o1[j + 1] = a11;
    }
    if (EPI == EPI_QKV && j >= p.D) {
      // scatter k / v of the current token into the cache at input_pos (fast_model.py:111-112)
      const int which = (j - p.D) / p.D;  // 0 = k, 1 = v
      const int jj = (j - p.D) - which * p.D;
      const int head = jj >> 7, d = jj & 127;
      const int pos = st.pos[u];
      const size_t e0 = (((size_t)r0 * p.H + head) * p.S_max + pos) * 128 + d;
      const size_t e1 = e0 + (size_t)p.H * p.S_max * 128;
      void* base = which ? p.vcache : p.kcache;
      if (p.kv_fp32) {
        float* c = reinterpret_cast<float*>(base);
        c[e0] = a00;
        c[e0 + 1] = a10;
        c[e1] = a01;
        c[e1 + 1] = a11;
      } else {
        __nv_bfloat16* c = reinterpret_cast<__nv_bfloat16*>(base);
        *reinterpret_cast<__nv_bfloat162*>(c + e0) = __floats2bfloat162_rn(a00, a10);
        *reinterpret_cast<__nv_bfloat162*>(c + e1) = __floats2bfloat162_rn(a01, a11);
      }
    }
  }
}

template <int EPI, bool LAYER = false, bool BIASED = false>
__global__ void __launch_bounds__(256, 2) k_gemv(GemvP p, S1State st) {
  extern __shared__ float xs[];  // [2][K] permuted
  __shared__ float red[16];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = p.K;
  const int n_items = (EPI == EPI_SWIGLU) ? p.M : (p.M >> 1);
  const int nwarps = gridDim.x * 8;
  const int KIT = K >> 8;
  pdl_launch_dependents();
  pdl_wait();  // activations written by the previous kernel are now visible

  const int u = st.slot_map[blockIdx.y];
  gemv_prologue<LAYER>(p, 2 * u, xs, red, [](int k) { return xs_perm(k); });

  // ---- main: each warp streams two weight rows at a time
  for (int item = blockIdx.x * 8 + warp; item < n_items; item += nwarps) {
    const uint4 *wa, *wb;
    gemv_rows<EPI>(p, item, lane, wa, wb);
    float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;  // [weight row][activation row]
#pragma unroll 4
    for (int it = 0; it < KIT; ++it) {
      const uint4 va = ldg_stream(wa + it * 32);
      const uint4 vb = ldg_stream(wb + it * 32);
      const float4* xp = reinterpret_cast<const float4*>(xs + it * 256);
      const float4* xq = reinterpret_cast<const float4*>(xs + K + it * 256);
      const float4 x0a = xp[lane], x0b = xp[32 + lane];
      const float4 x1a = xq[lane], x1b = xq[32 + lane];
      fma8(a00, va, x0a, x0b);
      fma8(a01, va, x1a, x1b);
      fma8(a10, vb, x0a, x0b);
      fma8(a11, vb, x1a, x1b);
    }
    a00 = warp_sum(a00);
    a01 = warp_sum(a01);
    a10 = warp_sum(a10);
    a11 = warp_sum(a11);
    if (lane == 0) gemv_epilogue<EPI, BIASED>(p, st, u, item, a00, a01, a10, a11);
  }
}

// ---------------------------------------------------------------------------------------------
// Shared by the int4, int8 and fp8 kernels (gemv_w4.cuh, gemv_w8.cuh, gemv_f8.cuh).
// Hint: bring [p, p + bytes) into L2 (one bulk request; the range is trimmed to whole 16-byte units inside it).
__device__ __forceinline__ void l2_prefetch(const void* p, size_t bytes) {
  const size_t a = reinterpret_cast<size_t>(p), lo = (a + 15) & ~(size_t)15, hi = (a + bytes) & ~(size_t)15;
  if (hi > lo)
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(lo), "r"((unsigned)(hi - lo)) : "memory");
}

// Up to five quantised matrices (one layer's wqkv, wo, w1, w3, w2, or lm_head / speaker_cond_pos once at create) and their
// bf16 row-major [M, K] destinations: the batch k_w4_dequant, k_w8_widen and k_f8_widen turn into tensor-core GEMM operands.
struct WidenBatch {
  const uint8_t* src[5];
  __nv_bfloat16* dst[5];
  int M[5], K[5];
  int n;
};

// ---------------------------------------------------------------------------------------------
// Decode attention: softmax(q K^T / sqrt(128) + causal mask) V over cache slots [0, pos]
// (fast_model.py:220-224 with the mask row of :148,151).  The reference attends to all 2048 slots
// through a boolean mask; masked slots carry exactly zero weight, so reading only [0, pos] is
// the same arithmetic on 393,216*L bytes instead of 805 MB (SURVEY.md D5).
// Split-KV flash decoding: grid (head, row, split); the last-arriving split merges.
constexpr int ATT_SPLITS = 8;

// Path B: arbitrary activation rows (batched decode rows or the 2*S rows of a prefill chunk); each row
// names its cache row and its own position, i.e. causal attention over [0, pos[row]].
struct RowsDev {
  int* cache_row;
  int* pos;
  int* tok;
  int* utt;
  int* cond;
};

template <bool KV_FP32>
__device__ __forceinline__ void load8(const void* base, size_t elem, float (&v)[8]) {
  if (KV_FP32) {
    const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem);
    const float4 a = __ldcg(p), b = __ldcg(p + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    const uint4 w = __ldcg(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(base) + elem));
    v[0] = bf_lo(w.x); v[1] = bf_hi(w.x); v[2] = bf_lo(w.y); v[3] = bf_hi(w.y);
    v[4] = bf_lo(w.z); v[5] = bf_hi(w.z); v[6] = bf_lo(w.w); v[7] = bf_hi(w.w);
  }
}

// ---------------------------------------------------------------------------------------------
// fp8 KV cache (MVB_KV_FP8, layout in include/mvb200.h): e4m3 codes where the bf16 cache has its elements, and one bf16
// scale per (layer, K|V, cache row, head, pos) in a region after all the codes.  Each new 128-element k or v -- the fp32
// qkv output exactly as the projection produced it -- is stored as
//   s = bf16_rn(max(amax|x| / 448, FLT_EPSILON)),   q = e4m3_rn(clamp(x / s, -448, 448))
// (mvb200/quantize.py quantize_kv_fp8); s q is exact in fp32 (8 + 4 significant bits), so attention runs the fp32-cache
// arithmetic over exact dequantised values.  Non-finite input: a NaN anywhere in x gives s = NaN (bits 0x7fc0) and every
// code 0x7f; otherwise +-inf makes s = +inf, its own code 0x7f (inf / inf) and every finite element's code a signed zero.
enum { KVC_BF16 = 0, KVC_FP32 = 1, KVC_FP8 = 2 };   // cache formats, == MVB_KV_*

struct KvF8 {
  uint8_t* kc;           // this layer's K codes [rows][H][S_max][128]
  uint8_t* vc;           // V codes
  __nv_bfloat16* ks;     // K scales [rows][H][S_max]
  __nv_bfloat16* vs;     // V scales
};

// e4m3 code of one quotient r = x / s: NaN -> 0x7f, else round to nearest even after the clamp (the hardware cvt)
__device__ __forceinline__ uint32_t kv_f8_code(float r) {
  if (r != r) return 0x7fu;
  return __nv_cvt_float_to_fp8(fminf(fmaxf(r, -448.f), 448.f), __NV_SATFINITE, __NV_E4M3);
}

// One warp per (activation row n, head, K|V): a float4 per lane, the amax as an unsigned max over |x|'s bit patterns (a NaN
// sorts above +inf, where fmaxf would drop it), one 128-byte store of codes, one scale store.  ROWS: row n of qkv goes to
// cache row rw.cache_row[n] at rw.pos[n] (path B: prefill chunks and batched decode); else row n is CFG row n & 1 of slot
// u = st.slot_map[n >> 1], i.e. qkv / cache row 2u + (n & 1) at st.pos[u] (path A).
template <bool ROWS>
__global__ void __launch_bounds__(256) k_kv_store_f8(S1State st, RowsDev rw, int n_rows, const float* __restrict__ qkv,
                                                     KvF8 kv, int H, int S_max, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (gw >= n_rows * H * 2) return;
  const int which = gw & 1, h = (gw >> 1) % H, n = (gw >> 1) / H;
  int row, cache_row, pos;
  if (ROWS) {
    row = n;
    cache_row = rw.cache_row[n];
    pos = rw.pos[n];
  } else {
    const int u = st.slot_map[n >> 1];
    row = cache_row = 2 * u + (n & 1);
    pos = st.pos[u];
  }
  const float4 x = *reinterpret_cast<const float4*>(qkv + (size_t)row * 3 * D + (size_t)(1 + which) * D + h * 128 + lane * 4);
  const unsigned m = max(max(__float_as_uint(x.x) & 0x7fffffffu, __float_as_uint(x.y) & 0x7fffffffu),
                         max(__float_as_uint(x.z) & 0x7fffffffu, __float_as_uint(x.w) & 0x7fffffffu));
  const unsigned amax = __reduce_max_sync(0xffffffffu, m);
  uint32_t codes = 0x7f7f7f7fu;
  __nv_bfloat16 sb = __ushort_as_bfloat16((unsigned short)0x7fc0);
  if (amax <= 0x7f800000u) {   // no NaN
    sb = __float2bfloat16_rn(fmaxf(__uint_as_float(amax) / 448.f, 1.1920928955078125e-7f));   // FLT_EPSILON
    const float s = __bfloat162float(sb);
    codes = kv_f8_code(x.x / s) | kv_f8_code(x.y / s) << 8 | kv_f8_code(x.z / s) << 16 | kv_f8_code(x.w / s) << 24;
  }
  const size_t slot = ((size_t)cache_row * H + h) * S_max + pos;
  reinterpret_cast<uint32_t*>(which ? kv.vc : kv.kc)[slot * 32 + lane] = codes;
  if (lane == 0) (which ? kv.vs : kv.ks)[slot] = sb;
}

// 8 codes of one position (8 bytes per lane: a 128-byte line per half-warp) times the position's scale, exactly
// (hardware e4m3x2 -> f16x2 conversion, then one fp32 product with 12 significant bits)
__device__ __forceinline__ void load8_f8(const uint8_t* codes, size_t elem, float scale, float (&v)[8]) {
  const uint2 w = __ldcg(reinterpret_cast<const uint2*>(codes + elem));
  const uint32_t wd[2] = {w.x, w.y};
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(wd[j] >> (16 * i)), __NV_E4M3);
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
      v[4 * j + 2 * i] = f.x * scale;
      v[4 * j + 2 * i + 1] = f.y * scale;
    }
}

// One (query row, head, KV split): q = query vector (fp32, 128), cache_row/L select the K/V slice,
// pidx indexes the per-(row, head) partial slots, `ticket` is that pair's arrival counter.  KV: the cache's KVC_* format;
// kscale / vscale are an fp8 cache's scales (unused otherwise).
template <int KV>
__device__ __forceinline__ void attn_core(const float* __restrict__ qvec, const void* kcache, const void* vcache,
                                          int cache_row, int L, int h, int split, int H, int S_max,
                                          float* __restrict__ part_o, float* __restrict__ part_ml, size_t pair,
                                          unsigned* ticket, float* __restrict__ out_vec,
                                          const __nv_bfloat16* kscale = nullptr, const __nv_bfloat16* vscale = nullptr) {
  __shared__ float sm_o[8][128];
  __shared__ float sm_m[8], sm_l[8];
  __shared__ int sm_last;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, half = lane >> 4, sub = lane & 15;
  const int chunk = (((L + ATT_SPLITS - 1) / ATT_SPLITS) + 7) & ~7;
  const int start = split * chunk;
  const int end = min(L, start + chunk);

  float q[8];
  {
    const float scale = 0.08838834764831845f;  // 1/sqrt(128)
#pragma unroll
    for (int i = 0; i < 8; ++i) q[i] = qvec[sub * 8 + i] * scale;
  }
  const size_t row_base = ((size_t)cache_row * H + h) * S_max * 128 + sub * 8;
  const size_t scale_base = ((size_t)cache_row * H + h) * S_max;
  float m = -INFINITY, l = 0.f, o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = 0.f;

  for (int pb = start + warp * 2; pb < end; pb += 8) {
    const int p = pb + half;
    const bool valid = p < end;
    float kv[8];
    float s = 0.f;
    if (valid) {
      if constexpr (KV == KVC_FP8)
        load8_f8(reinterpret_cast<const uint8_t*>(kcache), row_base + (size_t)p * 128, bf16_to_f32(kscale[scale_base + p]), kv);
      else
        load8<KV == KVC_FP32>(kcache, row_base + (size_t)p * 128, kv);
#pragma unroll
      for (int i = 0; i < 8; ++i) s = fmaf(q[i], kv[i], s);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 8);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    if (valid) {
      if constexpr (KV == KVC_FP8)
        load8_f8(reinterpret_cast<const uint8_t*>(vcache), row_base + (size_t)p * 128, bf16_to_f32(vscale[scale_base + p]), kv);
      else
        load8<KV == KVC_FP32>(vcache, row_base + (size_t)p * 128, kv);
      const float mn = fmaxf(m, s);
      const float corr = __expf(m - mn);  // m = -inf on the first visit -> 0
      const float pw = __expf(s - mn);
      l = l * corr + pw;
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = o[i] * corr + pw * kv[i];
      m = mn;
    }
  }
  const int g = warp * 2 + half;
  if (sub == 0) {
    sm_m[g] = m;
    sm_l[g] = l;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) sm_o[g][sub * 8 + i] = o[i];
  __syncthreads();

  const size_t pidx = pair * ATT_SPLITS + split;
  {
    float M = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) M = fmaxf(M, sm_m[i]);
    float Ls = 0.f, O = 0.f;
    if (M > -INFINITY) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float w = __expf(sm_m[i] - M);
        Ls += sm_l[i] * w;
        O += sm_o[i][tid] * w;
      }
    }
    part_o[pidx * 128 + tid] = O;
    if (tid == 0) {
      part_ml[pidx * 2] = M;
      part_ml[pidx * 2 + 1] = Ls;
    }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned t = atomicAdd(ticket, 1u);
    sm_last = (t == ATT_SPLITS - 1);
  }
  __syncthreads();
  if (sm_last) {
    __threadfence();
    const size_t b = pair * ATT_SPLITS;
    float M = -INFINITY;
#pragma unroll
    for (int i = 0; i < ATT_SPLITS; ++i) M = fmaxf(M, __ldcg(part_ml + (b + i) * 2));
    float Ls = 0.f, O = 0.f;
#pragma unroll
    for (int i = 0; i < ATT_SPLITS; ++i) {
      const float mi = __ldcg(part_ml + (b + i) * 2);
      if (mi > -INFINITY) {
        const float w = __expf(mi - M);
        Ls += __ldcg(part_ml + (b + i) * 2 + 1) * w;
        O += __ldcg(part_o + (b + i) * 128 + tid) * w;
      }
    }
    out_vec[tid] = O / Ls;
    if (tid == 0) *ticket = 0u;
  }
}

// Path A: the two CFG rows of each utterance, positions from the decode state.
template <bool KV_FP32>
__global__ void __launch_bounds__(128) k_attn_decode(S1State st, const float* __restrict__ qkv, const void* kcache,
                                                     const void* vcache, float* __restrict__ part_o,
                                                     float* __restrict__ part_ml, float* __restrict__ out, int H,
                                                     int S_max, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int h = blockIdx.x, split = blockIdx.z;
  const int u = st.slot_map[blockIdx.y >> 1];
  const int r = 2 * u + (blockIdx.y & 1);
  attn_core<KV_FP32 ? KVC_FP32 : KVC_BF16>(qkv + (size_t)r * 3 * D + h * 128, kcache, vcache, r, st.pos[u] + 1, h, split, H,
                                         S_max, part_o, part_ml, (size_t)r * H + h, &st.attn_ticket[r * H + h],
                                         out + (size_t)r * D + h * 128);
}

// k_attn_decode over an fp8 cache
__global__ void __launch_bounds__(128) k_attn_decode_f8(S1State st, const float* __restrict__ qkv, KvF8 kv,
                                                        float* __restrict__ part_o, float* __restrict__ part_ml,
                                                        float* __restrict__ out, int H, int S_max, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int h = blockIdx.x, split = blockIdx.z;
  const int u = st.slot_map[blockIdx.y >> 1];
  const int r = 2 * u + (blockIdx.y & 1);
  attn_core<KVC_FP8>(qkv + (size_t)r * 3 * D + h * 128, kv.kc, kv.vc, r, st.pos[u] + 1, h, split, H, S_max, part_o, part_ml,
                    (size_t)r * H + h, &st.attn_ticket[r * H + h], out + (size_t)r * D + h * 128, kv.ks, kv.vs);
}

template <bool KV_FP32>
__global__ void __launch_bounds__(128) k_attn_rows(RowsDev rw, const float* __restrict__ qkv, const void* kcache,
                                                   const void* vcache, float* __restrict__ part_o,
                                                   float* __restrict__ part_ml, unsigned* tickets,
                                                   float* __restrict__ out, int H, int S_max, int D) {
  const int h = blockIdx.x, n = blockIdx.y, split = blockIdx.z;
  attn_core<KV_FP32 ? KVC_FP32 : KVC_BF16>(qkv + (size_t)n * 3 * D + h * 128, kcache, vcache, rw.cache_row[n], rw.pos[n] + 1,
                                         h, split, H, S_max, part_o, part_ml, (size_t)n * H + h, &tickets[n * H + h],
                                         out + (size_t)n * D + h * 128);
}

// k_attn_rows over an fp8 cache
__global__ void __launch_bounds__(128) k_attn_rows_f8(RowsDev rw, const float* __restrict__ qkv, KvF8 kv,
                                                      float* __restrict__ part_o, float* __restrict__ part_ml,
                                                      unsigned* tickets, float* __restrict__ out, int H, int S_max, int D) {
  const int h = blockIdx.x, n = blockIdx.y, split = blockIdx.z;
  attn_core<KVC_FP8>(qkv + (size_t)n * 3 * D + h * 128, kv.kc, kv.vc, rw.cache_row[n], rw.pos[n] + 1, h, split, H, S_max,
                    part_o, part_ml, (size_t)n * H + h, &tickets[n * H + h], out + (size_t)n * D + h * 128, kv.ks, kv.vs);
}

__global__ void k_rows_decode(S1State st, RowsDev rw, int n_utts) {
  const int r = threadIdx.x;
  if (r < 2 * n_utts) {
    const int u = st.slot_map[r >> 1], c = r & 1;
    rw.cache_row[r] = 2 * u + c;
    rw.pos[r] = st.pos[u];
    rw.tok[r] = st.row_tok[2 * u + c];
    rw.utt[r] = u;
    rw.cond[r] = (c == 0);
  }
}

// rows of one prefill chunk: n = c * Sc + s  <->  (CFG row c, token s0 + s of idx[2, S])
__global__ void k_rows_prefill(RowsDev rw, int utt, const int* __restrict__ idx, int S, int s0, int Sc, int pos0) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n < 2 * Sc) {
    const int c = n / Sc, s = n - c * Sc;
    rw.cache_row[n] = 2 * utt + c;
    rw.pos[n] = pos0 + s0 + s;
    rw.tok[n] = idx[c * S + s0 + s];
    rw.utt[n] = utt;
    rw.cond[n] = (c == 0);
  }
}

__global__ void __launch_bounds__(256) k_embed_rows(RowsDev rw, const __nv_bfloat16* __restrict__ tok_emb,
                                                    const __nv_bfloat16* __restrict__ pos_emb,
                                                    const float* __restrict__ spk_proj, float* __restrict__ x, int D) {
  const int n = blockIdx.x;
  const __nv_bfloat16* te = tok_emb + (size_t)rw.tok[n] * D;
  const __nv_bfloat16* pe = pos_emb + (size_t)rw.pos[n] * D;
  const bool cond = rw.cond[n] != 0;
  const float* sp = spk_proj + (size_t)rw.utt[n] * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float v = bf16_to_f32(te[d]) + bf16_to_f32(pe[d]);
    if (cond) v += sp[d];
    x[(size_t)n * D + d] = v;
  }
}

// gather the two last-position rows of a prefill chunk (n = Sc-1 and 2*Sc-1) into rows {0, 1}
__global__ void k_gather_last(const float* __restrict__ x, float* __restrict__ dst, int Sc, int D) {
  const int c = blockIdx.x;
  const float* src = x + (size_t)(c * Sc + Sc - 1) * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) dst[(size_t)c * D + d] = src[d];
}

// ---------------------------------------------------------------------------------------------
// sample(): CFG mix, temperature, top-k, top-p (ascending sort, drop cum <= 1-p, keep the last),
// softmax, argmax(p / Exp(1))     (fast_inference_utils.py:61-120).  One CTA per utterance.
// `decode_mode` additionally performs the loop bookkeeping of decode_n_tokens / generate
// (utils:160-172, 212-226): append, feed back, bump position, latch end-of-audio.
//
// Prompt guidance (mixins/causal.py:89-105, 224-262): a guided primary u with companion slot c mixes three rows,
// cond 2u, uncond-speaker 2u + 1 and uncond-prompt 2c, as (s + p - 1) cond + (1 - s) uncond_spk + (1 - p) uncond_prompt,
// then runs the same tail.  In decode mode the primary also does the companion's bookkeeping (the companion is fed
// `fed > end_of_audio ? end_of_text : fed`, causal.py:262) and hands back all four of its rows zeroed; the companion's
// own CTA does nothing.
constexpr int SAMP_THREADS = 1024;
constexpr int SAMP_PAD = 4096;

struct SampleP {
  const float* logits;  // [rows, V] (decode mode: engine logits buffer) or [2, V] / guided [3, V] (API mode)
  int V;
  int decode_mode;
  // API mode
  SamplingDev sp;
  float prompt_guidance;  // > 1: logits are [3, V] = {cond, uncond speaker, uncond prompt}
  const float* noise;
  unsigned long long step;
  int* token_out;
  float* probs_out;
  unsigned* grid_bar;  // decode mode: arrival counter of the persistent decode kernel, reset here between steps
};

__global__ void __launch_bounds__(SAMP_THREADS) k_sample(SampleP p, S1State st) {
  __shared__ float key[SAMP_PAD];
  __shared__ unsigned short sid[SAMP_PAD];
  __shared__ float wsum[32];
  __shared__ float s_bcast[4];
  __shared__ unsigned long long s_best[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int V = p.V;
  pdl_launch_dependents();   // the next decode kernel may start prefetching weights while we sample
  pdl_wait();                // logits of this step are complete
  if (p.decode_mode && p.grid_bar && blockIdx.x == 0 && tid == 0) *p.grid_bar = 0u;
  int u = 0;
  SamplingDev sp = p.sp;
  const float* noise = p.noise;
  unsigned long long step = p.step;
  const float* lc = p.logits;
  const float* lp = nullptr;     // uncond-prompt row of a guided utterance
  float pg = p.prompt_guidance;
  int comp = -1, eot = 0;        // decode mode: companion slot of a guided primary and its end_of_text token
  if (p.decode_mode) {
    u = st.slot_map[blockIdx.x];
    lc = p.logits + (size_t)(2 * u) * V;
    const int link = st.samp[u].link;
    if (link < 0) return;        // a companion: its primary reads, zeroes and advances its rows
    comp = link - 1;
    if (st.done[u]) {
      // a finished utterance still rides along in the batch (its rows are recomputed at a frozen position): hand its
      // logits rows back zeroed so the persistent kernel's red.add accumulation starts from zero every step
      float* z = const_cast<float*>(lc);
      for (int v = tid; v < 2 * V; v += SAMP_THREADS) z[v] = 0.f;
      if (comp >= 0) {   // and so are its companion's
        z = const_cast<float*>(p.logits) + (size_t)(2 * comp) * V;
        for (int v = tid; v < 2 * V; v += SAMP_THREADS) z[v] = 0.f;
      }
      return;
    }
    sp = st.samp[u];
    step = (unsigned long long)st.n_gen[u];
    noise = st.noise[u] ? st.noise[u] + (size_t)(st.n_gen[u] - st.noise_base[u]) * V : nullptr;
    if (comp >= 0) {
      const SamplingDev cs = st.samp[comp];
      pg = cs.guidance;
      eot = cs.end_of_audio;
      lp = p.logits + (size_t)(2 * comp) * V;
    }
  } else if (pg > 1.0f) {
    lp = lc + 2 * V;
  }
  const float* lu = lc + V;

  // -- CFG mix and temperature, with torch's rounding order (utils:116, :92)
  const float tdiv = fmaxf(sp.temperature, 1e-5f);
  if (lp == nullptr) {
    const float g = sp.guidance, omg = __fsub_rn(1.0f, sp.guidance);
    for (int v = tid; v < SAMP_PAD; v += SAMP_THREADS) {
      float k = INFINITY;
      if (v < V) k = __fdiv_rn(__fadd_rn(__fmul_rn(g, lc[v]), __fmul_rn(omg, lu[v])), tdiv);
      key[v] = k;
      sid[v] = (unsigned short)v;
    }
  } else {
    // causal.py:100-104 with Python-float coefficients: each formed in double and rounded once to fp32, as torch does
    // for a Python scalar times an fp32 tensor; then ((base c + (1-s) u) + (1-p) up).  s and p arrive through the C ABI
    // already rounded to fp32, so for a scale fp32 cannot represent a coefficient can differ from torch's by half an ulp
    // of that scale plus its own rounding (1 ulp at (3.1, 1.7), 3 ulps of 1 - s at s = 1.1); dyadic scales are exact.
    const double s = sp.guidance, pd = pg;
    const float cb = __double2float_rn(s + pd - 1.0), cs = __double2float_rn(1.0 - s), cp = __double2float_rn(1.0 - pd);
    for (int v = tid; v < SAMP_PAD; v += SAMP_THREADS) {
      float k = INFINITY;
      if (v < V)
        k = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(cb, lc[v]), __fmul_rn(cs, lu[v])), __fmul_rn(cp, lp[v])), tdiv);
      key[v] = k;
      sid[v] = (unsigned short)v;
    }
  }
  __syncthreads();
  if (p.decode_mode) {
    // the persistent decode kernel accumulates split-K partial logits with red.add: hand the rows back zeroed
    // (after the barrier: every thread has consumed its logits by now)
    float* z = const_cast<float*>(lc);
    for (int v = tid; v < 2 * V; v += SAMP_THREADS) z[v] = 0.f;
    if (comp >= 0) {
      z = const_cast<float*>(lp);
      for (int v = tid; v < 2 * V; v += SAMP_THREADS) z[v] = 0.f;
    }
  }

  // -- ascending bitonic sort of (logit, index); padding (+inf) sinks to the end
  for (int k = 2; k <= SAMP_PAD; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < SAMP_PAD / 2; t += SAMP_THREADS) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int ixj = i | j;
        const bool up = ((i & k) == 0);
        const float a = key[i], b = key[ixj];
        const unsigned short ia = sid[i], ib = sid[ixj];
        const bool gt = (a > b) || (a == b && ia > ib);
        if (gt == up) {
          key[i] = b; key[ixj] = a;
          sid[i] = ib; sid[ixj] = ia;
        }
      }
      // strides <= 32: a warp's 32 pair slots (and the second batch at +SAMP_THREADS) stay inside its own two
      // 64-element blocks for all of j = 32 .. 1, so consecutive warp-local stages only need a warp barrier
      // (27 block barriers instead of 78 for 4096 keys)
      const int nj = (j > 1) ? (j >> 1) : k;   // stride of the next stage
      if (j > 32 || nj > 32) __syncthreads();
      else __syncwarp();
    }
  }

  // -- top-k: logits < (k-th largest) -> -inf (utils:94-97)
  if (sp.top_k > 0) {
    const int kk = min(sp.top_k, V);
    const float pivot = key[V - kk];
    __syncthreads();
    for (int i = tid; i < V; i += SAMP_THREADS)
      if (key[i] < pivot) key[i] = -INFINITY;
    __syncthreads();
  }

  // -- softmax over the sorted logits, inclusive cumulative sum (utils:72)
  const float mx = key[V - 1];
  float e[4];
  float loc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = tid * 4 + i;
    e[i] = (idx < V) ? expf(key[idx] - mx) : 0.f;
    loc += e[i];
  }
  // block inclusive scan of per-thread totals
  float incl = loc;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    float w = wsum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float n = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += n;
    }
    wsum[lane] = w;
  }
  __syncthreads();
  const float total = wsum[31];
  const float before = (warp ? wsum[warp - 1] : 0.f) + (incl - loc);

  // -- top-p: drop sorted entries whose cumulative probability <= 1 - top_p, never the last (utils:75-77)
  float kept_sum_loc = 0.f;
  {
    const bool use_p = sp.top_p > 0.f;
    const float thr = __fsub_rn(1.0f, sp.top_p);
    float run = before;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid * 4 + i;
      run += e[i];
      if (idx < V) {
        const float cum = run / total;
        bool drop = use_p && (cum <= thr) && (idx != V - 1);
        if (key[idx] == -INFINITY) drop = true;
        if (drop) e[i] = 0.f;
        kept_sum_loc += e[i];
      }
    }
  }
  __syncthreads();  // everyone has read key[]/wsum[] -> reuse key[] for the un-sorted probabilities
  float ks = warp_sum(kept_sum_loc);
  if (lane == 0) wsum[warp] = ks;
  // scatter kept exp-values back to vocabulary order (utils:80-81)
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = tid * 4 + i;
    if (idx < V) key[SAMP_PAD - 1 - sid[idx]] = e[i];  // reversed addressing: never collides with unread sorted slots
  }
  __syncthreads();
  if (warp == 0) {
    float w = warp_sum(wsum[lane]);
    if (lane == 0) s_bcast[0] = w;
  }
  __syncthreads();
  const float kept_total = s_bcast[0];

  // -- probs = softmax(masked logits); token = argmax(probs / q)   (utils:101, :61-65)
  unsigned long long best = 0ull;
  for (int v = tid; v < V; v += SAMP_THREADS) {
    const float pr = key[SAMP_PAD - 1 - v] / kept_total;
    if (p.probs_out && !p.decode_mode) p.probs_out[v] = pr;
    float qv;
    if (noise) {
      qv = noise[v];
    } else {
      const uint4 rnd = philox4x32_10(make_uint4((unsigned)v, (unsigned)step, (unsigned)(step >> 32), (unsigned)u),
                                      make_uint2((unsigned)sp.seed, (unsigned)(sp.seed >> 32)));
      qv = philox_exp1(rnd.x);
    }
    const float score = __fdiv_rn(pr, qv);
    // order-preserving key for non-negative floats; ties resolve to the lowest index like torch.argmax
    const unsigned long long cand =
        ((unsigned long long)__float_as_uint(score) << 32) | (unsigned long long)(0xffffffffu - (unsigned)v);
    best = cand > best ? cand : best;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long n = __shfl_xor_sync(0xffffffffu, best, o);
    best = n > best ? n : best;
  }
  if (lane == 0) s_best[warp] = best;
  __syncthreads();
  if (warp == 0) {
    best = s_best[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long n = __shfl_xor_sync(0xffffffffu, best, o);
      best = n > best ? n : best;
    }
    if (lane == 0) {
      const int tok = (int)(0xffffffffu - (unsigned)(best & 0xffffffffull));
      if (!p.decode_mode) {
        *p.token_out = tok;
      } else {
        const int n = st.n_gen[u];
        int fed = tok;
        if (st.forced[u]) fed = st.forced[u][n];
        st.sampled_tokens[(size_t)u * st.max_new + n] = tok;
        st.gen_tokens[(size_t)u * st.max_new + n] = fed;
        st.row_tok[2 * u] = fed;
        st.row_tok[2 * u + 1] = fed;
        // Latch termination (utils:161 EOA; utils:196-204 token budget; context end) and keep the position inside the
        // cache: a finished utterance is re-run at its last valid slot while the rest of the batch continues, so no
        // body ever reads pos_emb[block_size] or appends K/V past slot block_size - 1.
        const int np = st.pos[u] + 1;
        const bool stop = fed == sp.end_of_audio || np >= st.block_size || n + 1 >= st.max_new || n + 1 >= st.budget[u];
        if (!stop) st.pos[u] = np;
        st.n_gen[u] = n + 1;
        if (stop) st.done[u] = 1;
        if (comp >= 0) {   // the companion follows the primary's positions; text tokens reach it as end_of_text
          const int fc = fed > sp.end_of_audio ? eot : fed;
          st.sampled_tokens[(size_t)comp * st.max_new + n] = tok;
          st.gen_tokens[(size_t)comp * st.max_new + n] = fc;
          st.row_tok[2 * comp] = fc;
          st.row_tok[2 * comp + 1] = fc;
          if (!stop) st.pos[comp] = np;
          st.n_gen[comp] = n + 1;
          if (stop) st.done[comp] = 1;
        }
      }
    }
  }
}

}  // namespace mvb
