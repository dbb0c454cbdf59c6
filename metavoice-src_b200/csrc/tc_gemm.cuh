// Weight-streaming skinny GEMM on the tensor cores ("path B"): Y[n, j] = sum_k X[n, k] * W[j, k].
//
// The projection weights are the big operand (W[M, K] bf16, row-major = K-major), the activations the
// skinny one (R <= 128 rows), so the roles are swapped with respect to a textbook GEMM: a 128-row tile
// of W is the MMA "A" operand, the activation rows are the "B" operand.  Weights go HBM -> TMA ->
// 128B-swizzled shared memory -> ldmatrix -> mma.sync.m16n8k16 with fp32 accumulators in registers.
//
// Precision: weights are exactly bf16; activations are split x = hi + lo (two bf16 terms, 16 mantissa
// bits); the lo rows follow the hi rows in the B buffer and both products go into the same accumulator,
// so the product matches an fp32-activation GEMM to ~1e-5 while the MMA count stays irrelevant (the
// kernel is HBM-bound on W).
//
// Warp roles (288 threads, tc_mainloop): warp 0 = TMA producer, warps 1..8 = consumers; consumer w owns weight
// rows [16 (w - 1), 16 w) of the tile and every activation row, and runs the fused epilogue straight from its
// registers.  grid = (row tiles, K splits); split-K partial tiles go through a scratch buffer, every split
// of a tile reduces its share of the rows in a fixed order (deterministic), then applies the operator epilogue.
#pragma once
#include "tc.cuh"
#include "tc_gemm_host.cuh"

namespace mvb {

struct GemmP {
  int M, K;        // weight matrix [M, K]
  int NB;          // rows of the B buffer = Rpad * (1 + split_lo)
  int Rpad;        // rows reserved for the hi terms (multiple of 16, <= 128)
  int R;           // real activation rows (<= Rpad)
  int split_lo;    // 1: rows [Rpad, 2*Rpad) of B hold the lo terms
  int ksplit;      // gridDim.y
  int stages;      // smem ring depth
  float* scratch;  // [tiles][ksplit][(1 + swiglu) * Rpad][128] fp32 partial tiles (ksplit > 1)
  unsigned* tickets;  // [256]: arrivals per tile in [0, 128), completions per tile in [128, 256)
  float* out;
  int ldo;
  // G_QKV: KVCache.update scatter (fast_model.py:104-113)
  void* kcache;
  void* vcache;
  const int* row_cache;  // [R] cache row of each activation row
  const int* row_pos;    // [R] cache position of each activation row
  int H, S_max, D, kv_fp32;
  // bf16 [M] per-row vectors of W (and W3), applied once per output after the (split-K) sum: the row scales of int8
  // weights (the widened q, SCALED) or the Linear biases (GPTConfig bias=True, BIASED).  No instance uses both, so
  // they share the slots: a larger GemmP costs the existing instances registers.
  union { const __nv_bfloat16* scale; const __nv_bfloat16* bias; };
  union { const __nv_bfloat16* scale3; const __nv_bfloat16* bias3; };
};

constexpr int GEMM_THREADS = 288;

template <int EPI, bool SCALED, bool BIASED>
__device__ __forceinline__ void gemm_apply(const GemmP& p, int n, int j, float y, float y3) {
  if (SCALED) {
    y *= bf16_to_f32(p.scale[j]);
    if (EPI == G_SWIGLU) y3 *= bf16_to_f32(p.scale3[j]);
  }
  if (BIASED) {
    y += bf16_to_f32(p.bias[j]);
    if (EPI == G_SWIGLU) y3 += bf16_to_f32(p.bias3[j]);
  }
  if (EPI == G_STORE) {
    p.out[(size_t)n * p.ldo + j] = y;
  } else if (EPI == G_RESID) {
    p.out[(size_t)n * p.ldo + j] += y;
  } else if (EPI == G_SWIGLU) {
    p.out[(size_t)n * p.ldo + j] = (y / (1.f + expf(-y))) * y3;
  } else if (EPI == G_GELU) {   // nn.GELU(approximate='none'): the exact erf form
    p.out[(size_t)n * p.ldo + j] = 0.5f * y * (1.f + erff(y * (float)M_SQRT1_2));
  } else {
    p.out[(size_t)n * p.ldo + j] = y;
    if (j >= p.D) {
      const int which = (j - p.D) / p.D;
      const int jj = (j - p.D) - which * p.D;
      const int head = jj >> 7, d = jj & 127;
      const size_t e = (((size_t)p.row_cache[n] * p.H + head) * p.S_max + p.row_pos[n]) * 128 + d;
      void* base = which ? p.vcache : p.kcache;
      if (p.kv_fp32)
        reinterpret_cast<float*>(base)[e] = y;
      else
        reinterpret_cast<__nv_bfloat16*>(base)[e] = __float2bfloat16_rn(y);
    }
  }
}

// NC = n8 column chunks the accumulator holds (>= Rpad / 8; the chunks past Rpad / 8 are skipped at run time).
// SCALED: int8 weights, p.scale (p.scale3) multiply each output row after the sum; BIASED: p.bias (p.bias3) are added to
// it.  Both are template flags, so that the unscaled bias-free instances compile exactly as without them; no instance has
// both.
template <int EPI, int NC, bool SCALED, bool BIASED>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_tc_gemm(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA3,
          const __grid_constant__ CUtensorMap tmB, const GemmP p) {
  constexpr int NA = (EPI == G_SWIGLU) ? 2 : 1;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad_1024(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tile = blockIdx.x, split = blockIdx.y;
  const int nkb = p.K >> 6;
  const int kb0 = (int)(((long long)split * nkb) / p.ksplit);
  const int kb1 = (int)(((long long)(split + 1) * nkb) / p.ksplit);

  if (tid == 0) {
    ptx::prefetch_tensormap(&tmA);
    ptx::prefetch_tensormap(&tmB);
    if (NA == 2) ptx::prefetch_tensormap(&tmA3);
  }
  const uint64_t pol_w = ptx::policy_evict_first();  // weights are streamed exactly once per pass
  float acc[NA][NC][4];
  const bool consumer = tc_mainloop<NA, NC>(
      smem, p.stages, NA * GEMM_A_BYTES + p.NB * 128, NA * GEMM_A_BYTES, kb1 - kb0, p.Rpad >> 3, p.Rpad, p.split_lo,
      [&](int it, uint32_t st, uint32_t full) {
        const int kc = (kb0 + it) * 64;
        ptx::tma_load_2d_hint(st, &tmA, full, kc, tile * 128, pol_w);
        if (NA == 2) ptx::tma_load_2d_hint(st + GEMM_A_BYTES, &tmA3, full, kc, tile * 128, pol_w);
        ptx::tma_load_2d(st + NA * GEMM_A_BYTES, &tmB, full, kc, 0);
      },
      acc);
  if (!consumer) return;

  // ===== consumers: the epilogue straight from the accumulator registers =====
  const int ct = tid - 32;                 // 0..255
  const int w16 = 16 * (warp - 1);         // first weight row of this warp inside the tile
  const int nc = p.Rpad >> 3;
  // accumulator element e of chunk c: weight row w16 + (lane >> 2) + 8 (e >> 1), activation row 8 c + 2 (lane & 3) + (e & 1)
  const int rl0 = w16 + (lane >> 2), n0 = 2 * (lane & 3);
  if (p.ksplit == 1) {
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int n = 8 * c + n0 + (e & 1), j = tile * 128 + rl0 + 8 * (e >> 1);
        if (c < nc && n < p.R && j < p.M) gemm_apply<EPI, SCALED, BIASED>(p, n, j, acc[0][c][e], acc[NA - 1][c][e]);
      }
    return;
  }
  const int ncols = NA * p.Rpad;
  float* mine = p.scratch + ((size_t)(tile * p.ksplit + split) * ncols) * 128;
#pragma unroll
  for (int a = 0; a < NA; ++a)
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (c < nc) mine[(size_t)(a * p.Rpad + 8 * c + n0 + (e & 1)) * 128 + rl0 + 8 * (e >> 1)] = acc[a][c][e];
  __threadfence();
  asm volatile("bar.sync 1, 256;" ::: "memory");
  // Every split of this tile waits for all of them (grid = tiles x ksplit <= SM count: all co-resident), then reduces
  // ITS OWN share of the activation rows -- the reduction is spread over the ksplit CTAs instead of serialising
  // R x ksplit dependent L2 round trips in the last arriver.  The order of the sum over splits is fixed, so the result
  // stays run-to-run deterministic.
  if (ct == 0) {
    atomicAdd(&p.tickets[tile], 1u);
    wait_counter(p.tickets + tile, (unsigned)p.ksplit);
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  {
    const int row_local = ct & 127, j = tile * 128 + row_local;
    const int r_lo = (int)(((long long)split * p.R) / p.ksplit), r_hi = (int)(((long long)(split + 1) * p.R) / p.ksplit);
    const float* base = p.scratch + ((size_t)tile * p.ksplit * ncols) * 128 + row_local;
    for (int n = r_lo + (ct >> 7); n < r_hi; n += 2) {
      float y = 0.f, y3 = 0.f;
#pragma unroll 8
      for (int sp = 0; sp < p.ksplit; ++sp) {
        const float* ps = base + ((size_t)sp * ncols) * 128;
        y += __ldcg(ps + (size_t)n * 128);
        if (NA == 2) y3 += __ldcg(ps + (size_t)(p.Rpad + n) * 128);
      }
      if (j < p.M) gemm_apply<EPI, SCALED, BIASED>(p, n, j, y, y3);
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (ct == 0) {                          // the split that finishes last re-arms both counters for the next launch
    const unsigned t = atomicAdd(&p.tickets[128 + tile], 1u);
    if (t == (unsigned)p.ksplit - 1u) {
      p.tickets[128 + tile] = 0u;
      p.tickets[tile] = 0u;
    }
  }
}

// B-operand preparation: one CTA per activation row.  Optional norm, then the exact two-term bf16 split x = hi + lo.
//   LAYER = false: RMSNorm when gain != null (fast_model.py:250-261: fp32 statistics, then gain), else none.
//   LAYER = true : LayerNorm (layers/layers.py:8-17, F.layer_norm): fp32 mean, then the biased variance as a second pass
//                  over the centred row, (x - mean) * rsqrt(var + eps) * gain (+ beta when non-null); gain is required.
// A template flag, so that the RMS / no-norm instance stage 1 uses compiles exactly as without it.
template <bool LAYER>
static __global__ void __launch_bounds__(256) k_prep_b(const float* __restrict__ x, int ldx, const __nv_bfloat16* __restrict__ gain,
                                                const __nv_bfloat16* __restrict__ beta, float eps, int K, int Rpad, int R,
                                                int split_lo, __nv_bfloat16* __restrict__ B) {
  __shared__ float red[8];
  const int n = blockIdx.x, tid = threadIdx.x;
  if (n >= R) {  // padding rows [R, Rpad) of the B operand must read as zero
    const __nv_bfloat16 z = __float2bfloat16_rn(0.f);
    for (int k = tid; k < K; k += 256) {
      B[(size_t)n * K + k] = z;
      if (split_lo) B[(size_t)(Rpad + n) * K + k] = z;
    }
    return;
  }
  const float* xr = x + (size_t)n * ldx;
  if (LAYER) {
    float s = 0.f;
    for (int k = tid; k < K; k += 256) s += xr[k];
    s = warp_sum(s);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i];
    const float mean = t / (float)K;
    __syncthreads();                       // every thread has read red before it is reused
    float ss = 0.f;
    for (int k = tid; k < K; k += 256) {
      const float d = xr[k] - mean;
      ss = fmaf(d, d, ss);
    }
    ss = warp_sum(ss);
    if ((tid & 31) == 0) red[tid >> 5] = ss;
    __syncthreads();
    t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i];
    const float rs = rsqrtf(t / (float)K + eps);
    for (int k = tid; k < K; k += 256) {
      float v = ((xr[k] - mean) * rs) * bf16_to_f32(gain[k]);
      if (beta != nullptr) v += bf16_to_f32(beta[k]);
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      B[(size_t)n * K + k] = h;
      if (split_lo) B[(size_t)(Rpad + n) * K + k] = lo_term(v, h);
    }
    return;
  }
  float rs = 1.f;
  if (gain != nullptr) {
    float ss = 0.f;
    for (int k = tid; k < K; k += 256) {
      const float v = xr[k];
      ss = fmaf(v, v, ss);
    }
    ss = warp_sum(ss);
    if ((tid & 31) == 0) red[tid >> 5] = ss;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i];
    rs = rsqrtf(t / (float)K + eps);
  }
  for (int k = tid; k < K; k += 256) {
    float v = xr[k];
    if (gain != nullptr) v = (v * rs) * bf16_to_f32(gain[k]);
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    B[(size_t)n * K + k] = h;
    if (split_lo) B[(size_t)(Rpad + n) * K + k] = lo_term(v, h);
  }
}

}  // namespace mvb
