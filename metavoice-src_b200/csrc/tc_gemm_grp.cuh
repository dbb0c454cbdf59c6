// The weight-streaming GEMM of tc_gemm.cuh grouped over units that each bring their own weights: one launch, grid
// (row tiles, K splits, units).  Every activation row belongs to one unit (row_grp[n] -> g2u); the B operand holds all
// rows in their places, each normalised with its own unit's gain and beta (k_prep_b_grp), and a unit's CTAs store only
// the outputs of its own rows, so the epilogue writes every row where it is (out row n, cache row / position of row n).
// Used for a stage-1 decode batch whose slots are on different voices (stage1_engine.cu); the single-weight path
// (k_prep_b + k_tc_gemm) is untouched.
#pragma once
#include "tc_gemm.cuh"

namespace mvb {

struct GemmGrp {
  const int* row_grp;                                // [R] voice group of each activation row
  int g2u[GEMM_MAX_GROUPS];                          // voice group -> unit (blockIdx.z)
  const CUtensorMap* tmA[GEMM_MAX_GROUPS];           // per unit, in global memory: W (and W3 for SwiGLU)
  const CUtensorMap* tmA3[GEMM_MAX_GROUPS];
  const __nv_bfloat16* bias[GEMM_MAX_GROUPS];        // BIASED: per unit
  const __nv_bfloat16* bias3[GEMM_MAX_GROUPS];
};

template <int EPI, int NC, bool BIASED>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_tc_gemm_grp(const __grid_constant__ CUtensorMap tmB, const GemmP p, const GemmGrp q) {
  constexpr int NA = (EPI == G_SWIGLU) ? 2 : 1;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad_1024(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tile = blockIdx.x, split = blockIdx.y, unit = blockIdx.z;
  const int nkb = p.K >> 6;
  const int kb0 = (int)(((long long)split * nkb) / p.ksplit);
  const int kb1 = (int)(((long long)(split + 1) * nkb) / p.ksplit);
  const CUtensorMap* tA = q.tmA[unit];
  const CUtensorMap* tA3 = q.tmA3[unit];
  if (tid == 0) {
    ptx::prefetch_tensormap(tA);
    ptx::prefetch_tensormap(&tmB);
    if (NA == 2) ptx::prefetch_tensormap(tA3);
  }
  const uint64_t pol_w = ptx::policy_evict_first();
  float acc[NA][NC][4];
  const bool consumer = tc_mainloop<NA, NC>(
      smem, p.stages, NA * GEMM_A_BYTES + p.NB * 128, NA * GEMM_A_BYTES, kb1 - kb0, p.Rpad >> 3, p.Rpad, p.split_lo,
      [&](int it, uint32_t st, uint32_t full) {
        const int kc = (kb0 + it) * 64;
        ptx::tma_load_2d_hint(st, tA, full, kc, tile * 128, pol_w);
        if (NA == 2) ptx::tma_load_2d_hint(st + GEMM_A_BYTES, tA3, full, kc, tile * 128, pol_w);
        ptx::tma_load_2d(st + NA * GEMM_A_BYTES, &tmB, full, kc, 0);
      },
      acc);
  if (!consumer) return;

  GemmP pu = p;
  if (BIASED) { pu.bias = q.bias[unit]; pu.bias3 = q.bias3[unit]; }
  auto mine = [&](int n) { return q.g2u[q.row_grp[n]] == unit; };
  const int ct = tid - 32;
  const int w16 = 16 * (warp - 1);
  const int nc = p.Rpad >> 3;
  const int rl0 = w16 + (lane >> 2), n0 = 2 * (lane & 3);
  if (p.ksplit == 1) {
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int n = 8 * c + n0 + (e & 1), j = tile * 128 + rl0 + 8 * (e >> 1);
        if (c < nc && n < p.R && j < p.M && mine(n)) gemm_apply<EPI, false, BIASED>(pu, n, j, acc[0][c][e], acc[NA - 1][c][e]);
      }
    return;
  }
  // split-K: each unit has its own partial tiles and arrival counters (tiles x ksplit x units <= the SM count)
  const int ncols = NA * p.Rpad;
  const int tiles = gridDim.x;
  float* scratch = p.scratch + (size_t)unit * tiles * p.ksplit * ncols * 128;
  unsigned* tickets = p.tickets + (size_t)unit * 256;
  float* mine_s = scratch + ((size_t)(tile * p.ksplit + split) * ncols) * 128;
#pragma unroll
  for (int a = 0; a < NA; ++a)
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (c < nc) mine_s[(size_t)(a * p.Rpad + 8 * c + n0 + (e & 1)) * 128 + rl0 + 8 * (e >> 1)] = acc[a][c][e];
  __threadfence();
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (ct == 0) {
    atomicAdd(&tickets[tile], 1u);
    wait_counter(tickets + tile, (unsigned)p.ksplit);
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  {
    const int row_local = ct & 127, j = tile * 128 + row_local;
    const int r_lo = (int)(((long long)split * p.R) / p.ksplit), r_hi = (int)(((long long)(split + 1) * p.R) / p.ksplit);
    const float* base = scratch + ((size_t)tile * p.ksplit * ncols) * 128 + row_local;
    for (int n = r_lo + (ct >> 7); n < r_hi; n += 2) {
      if (!mine(n)) continue;
      float y = 0.f, y3 = 0.f;
#pragma unroll 8
      for (int sp = 0; sp < p.ksplit; ++sp) {
        const float* ps = base + ((size_t)sp * ncols) * 128;
        y += __ldcg(ps + (size_t)n * 128);
        if (NA == 2) y3 += __ldcg(ps + (size_t)(p.Rpad + n) * 128);
      }
      if (j < p.M) gemm_apply<EPI, false, BIASED>(pu, n, j, y, y3);
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (ct == 0) {
    const unsigned t = atomicAdd(&tickets[128 + tile], 1u);
    if (t == (unsigned)p.ksplit - 1u) {
      tickets[128 + tile] = 0u;
      tickets[tile] = 0u;
    }
  }
}

// k_prep_b with each row's own norm operands: gain[u] / beta[u] of its unit u = g2u[row_grp[n]] (all null: no norm).
struct PrepGrp {
  const int* row_grp;
  int g2u[GEMM_MAX_GROUPS];
  const __nv_bfloat16* gain[GEMM_MAX_GROUPS];
  const __nv_bfloat16* beta[GEMM_MAX_GROUPS];
};

template <bool LAYER>
static __global__ void __launch_bounds__(256) k_prep_b_grp(const float* __restrict__ x, int ldx, PrepGrp g, float eps, int K,
                                                    int Rpad, int R, int split_lo, __nv_bfloat16* __restrict__ B) {
  __shared__ float red[8];
  const int n = blockIdx.x, tid = threadIdx.x;
  if (n >= R) {
    const __nv_bfloat16 z = __float2bfloat16_rn(0.f);
    for (int k = tid; k < K; k += 256) {
      B[(size_t)n * K + k] = z;
      if (split_lo) B[(size_t)(Rpad + n) * K + k] = z;
    }
    return;
  }
  const int u = g.g2u[g.row_grp[n]];
  const __nv_bfloat16* gain = g.gain[u];
  const __nv_bfloat16* beta = g.beta[u];
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
    __syncthreads();
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
