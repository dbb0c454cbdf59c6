// Weight-only fp8 (e4m3) stage-1 kernels (quantisation_mode="fp8", an extension with no reference counterpart): the
// tensor-core decode GEMV that reads every weight byte once per step for all decoded slots (path A), and the per-layer
// widening that feeds the bf16 tensor-core GEMM for prefill and for batches of more than F8_MAX_UTTS slots (path B).
//
// fp8 matrix [M, K] (K % 256 == 0, M even; layout in include/mvb200.h, produced only by mvb200/quantize.py:pack_fp8_matrix):
//   M * K e4m3 codes in the fragment-native order of f8_code_offset, then at the next 256-byte boundary bf16 [M] row
//   scales s -- the int8 matrix layout, so the arena checks, k_tc_gemm's SCALED epilogue and WidenBatch take it unchanged.
// Function (every kernel): y_j = s_j * sum_k x_k q_jk -- fp32 sums over the exact e4m3 values, the scale applied once per
// output after the whole sum.
#pragma once
#include "stage1_kernels.cuh"
#include "gemv_w8.cuh"
#include "tc.cuh"

namespace mvb {

constexpr int F8_MAX_UTTS = 8;   // slots one k_gemv_f8 launch serves: 16 CFG rows, two n8 blocks of the MMA
constexpr int F8_IPC = 3;        // most 16-row blocks a CTA owns (the grid is sized so that none owns more)

// Byte offset of code (j, k) among the M * K codes.  Rows [0, M16), M16 = M & ~15, are cut into 16-row blocks and each
// block's K into 32-wide chunks; chunk c of block b is 512 contiguous bytes at (b * K / 32 + c) * 512, in which lane
// l = 4 g + t of a warp owns 16 bytes: word 2 s + h (k-step s of the chunk, k half h) holds, byte by byte, (row g, k0),
// (row g + 8, k0), (row g, k0 + 1), (row g + 8, k0 + 1) with k0 = 16 s + 8 h + 2 t -- the A fragment of
// mma.m16n8k16 for k-step s, so one 128-bit load gives a lane two k-steps.  Rows [M16, M) follow row-major.
__host__ __device__ inline size_t f8_code_offset(int j, int k, int M, int K) {
  const int M16 = M & ~15;
  if (j >= M16) return (size_t)j * K + k;
  const int r = j & 15, kk = k & 31;
  const int lane = ((r & 7) << 2) | ((kk & 7) >> 1);
  const int word = ((kk >> 4) << 1) | ((kk >> 3) & 1);
  const int byte = ((kk & 1) << 1) | (r >> 3);
  return ((size_t)(j >> 4) * (K >> 5) + (k >> 5)) * 512 + lane * 16 + word * 4 + byte;
}

// The e4m3 codes at bits 8-15 and 24-31 of t -> bf16x2 (the code at bits 8-15 in the low half), exactly.  The sign goes to
// bf16's sign and the 7 exponent | mantissa bits under bf16's exponent LSBs, which reads as the value times 2^-120 (a
// zero exponent field as a bf16 subnormal); one bf16x2 multiply by 2^120 restores it.  mul.bf16x2 keeps subnormal inputs,
// so the 14 subnormal codes convert exactly too.  The NaN codes 0x7f / 0xff, which the quantiser never emits, read as
// +-480.
__device__ __forceinline__ uint32_t f8x2_bf16x2(uint32_t t) {
  const uint32_t b = (t & 0x80008000u) | ((t >> 4) & 0x07F007F0u);
  uint32_t r;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(b), "r"(0x7B807B80u));   // 0x7b80 = bf16 2^120
  return r;
}

// A fragments of k-step s from one lane's 16 code bytes (words 2 s and 2 s + 1).
__device__ __forceinline__ void f8_frag(const uint4& w, int s, uint32_t (&a)[4]) {
  const uint32_t w0 = s ? w.z : w.x, w1 = s ? w.w : w.y;
  a[0] = f8x2_bf16x2(w0 << 8);   // row g,     k0, k0 + 1
  a[1] = f8x2_bf16x2(w0);        // row g + 8, k0, k0 + 1
  a[2] = f8x2_bf16x2(w1 << 8);   // row g,     k0 + 8, k0 + 9
  a[3] = f8x2_bf16x2(w1);        // row g + 8, k0 + 8, k0 + 9
}

// One lane's 16 bytes of chunk c of the partial block at rows [M16, M16 + nt) (row-major at `tail`), gathered into the
// fragment-native order; absent rows read as zero codes.
__device__ __forceinline__ uint4 f8_tail_chunk(const uint8_t* tail, int nt, int K, int c, int lane) {
  const int g = lane >> 2, t = lane & 3;
  uint32_t w[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int k0 = 32 * c + 16 * (q >> 1) + 8 * (q & 1) + 2 * t;
    const uint32_t lo = g < nt ? *reinterpret_cast<const uint16_t*>(tail + (size_t)g * K + k0) : 0u;
    const uint32_t hi = g + 8 < nt ? *reinterpret_cast<const uint16_t*>(tail + (size_t)(g + 8) * K + k0) : 0u;
    w[q] = __byte_perm(lo, hi, 0x5140);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// CTAs of a k_gemv_f8 launch over n_blocks 16-row blocks: one block per SM where there are enough, never more than
// F8_IPC blocks per CTA.  Depends on the shape and the SM count only, never on the number of slots.
__host__ __device__ inline int f8_gemv_ctas(int n_blocks, int n_sm) {
  const int one_per_sm = n_blocks < n_sm ? n_blocks : n_sm;
  const int need = (n_blocks + F8_IPC - 1) / F8_IPC;
  return need > one_per_sm ? need : one_per_sm;
}

// ---------------------------------------------------------------------------------------------
// k_gemv's contract (GemvP, RMSNorm when p.gain is set, the four epilogues) over fp8 matrices, for up to F8_MAX_UTTS
// slots in one launch: batch entries [8 y, 8 y + 8) of slot_map for blockIdx.y = y (gridDim.y = 1 up to 8 slots).
// CTA x owns the 16-row blocks x, x + G, ... (G = gridDim.x; for EPI_SWIGLU block b of w1 and of w3), so every weight byte
// is read once per launch.  Warp w owns the K range [w K / 8, (w + 1) K / 8), 32 k (one 16-byte load per lane per block)
// at a time, with the next chunk's weights and activations in flight while it multiplies the current one:
//   A = the weights, converted exactly to bf16 (f8_frag); B = the activation rows as bf16 hi and lo terms (tc.cuh
//   pack_hi_lo), column 2 i + c of n8 block NB = CFG row c of batch entry i; mma.m16n8k16 with fp32 accumulators, hi then
//   lo of each k-step into the same accumulator.
// The eight warps' sums are added in shared memory in warp order; RMSNorm's 1 / rms multiplies the sum (the activations
// enter the MMA times the gain only), then the row scale.  Every output column runs the same instructions whatever
// column it lands in, so a slot's outputs do not depend on the batch it is decoded in.  NB = 1 serves up to 4 slots.
template <int EPI, int NB>
__global__ void __launch_bounds__(256, 1) k_gemv_f8(GemvP p, S1State st, int n_utts) {
  constexpr int NM = EPI == EPI_SWIGLU ? 2 : 1;   // matrices per block: w1 and w3, or W
  __shared__ float red[8][NM][NB][128];
  __shared__ float ssq[8][NB * 8];
  __shared__ float rs[NB * 8];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int M = p.M, K = p.K;
  const int n_blocks = (M + 15) >> 4, M16 = M & ~15, G = gridDim.x;
  const uint8_t* Wq[NM];
  const __nv_bfloat16* Ws[NM];
  Wq[0] = reinterpret_cast<const uint8_t*>(p.W);
  if constexpr (NM == 2) Wq[1] = reinterpret_cast<const uint8_t*>(p.W3);
#pragma unroll
  for (int m = 0; m < NM; ++m) Ws[m] = reinterpret_cast<const __nv_bfloat16*>(Wq[m] + w8_scale_offset(M, K));
  const int n_mine = (int)blockIdx.x < n_blocks ? (n_blocks - 1 - (int)blockIdx.x) / G + 1 : 0;
  pdl_launch_dependents();
  if (warp == 0 && lane < F8_IPC * NM && lane / NM < n_mine) {   // the CTA's blocks, contiguous in the layout, into L2
    const int b = blockIdx.x + (lane / NM) * G;
    const int rows = M - 16 * b < 16 ? M - 16 * b : 16;
    l2_prefetch((lane % NM ? Wq[NM - 1] : Wq[0]) + (size_t)16 * b * K, (size_t)rows * K);
  }
  pdl_wait();  // activations written by the previous kernel are now visible

  const int e0 = 8 * blockIdx.y;                             // first batch entry of this launch row
  const int nu = n_utts - e0 < F8_MAX_UTTS ? n_utts - e0 : F8_MAX_UTTS;
  const float* xr[NB];                                       // activation row of this lane's B column in n8 block nb
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
    const int r = nb * 8 + g;
    xr[nb] = r < 2 * nu ? p.x + (size_t)(2 * st.slot_map[e0 + (r >> 1)] + (r & 1)) * p.ldx : nullptr;
  }
  const bool norm = p.gain != nullptr;
  const uint8_t* tail[NM];
#pragma unroll
  for (int m = 0; m < NM; ++m) tail[m] = Wq[m] + (size_t)M16 * K;
  const int nt = M - M16;

  auto load_w = [&](int c, uint4 (&w)[F8_IPC][NM]) {
#pragma unroll
    for (int i = 0; i < F8_IPC; ++i)
#pragma unroll
      for (int m = 0; m < NM; ++m) {
        const int b = blockIdx.x + i * G;
        if (i >= n_mine) w[i][m] = make_uint4(0, 0, 0, 0);
        else if (16 * b < M16) w[i][m] = ldg_stream(Wq[m] + ((size_t)b * (K >> 5) + c) * 512 + lane * 16);
        else w[i][m] = f8_tail_chunk(tail[m], nt, K, c, lane);
      }
  };
  // this lane's 8 activations of chunk c in n8 block nb: k = 32 c + 16 s + 2 t + {0, 1, 8, 9} for s = 0, 1
  auto load_x = [&](int c, float2 (&v)[NB][4]) {
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int k = 32 * c + 16 * (q >> 1) + 8 * (q & 1) + 2 * t;
        v[nb][q] = xr[nb] ? __ldcg(reinterpret_cast<const float2*>(xr[nb] + k)) : make_float2(0.f, 0.f);
      }
  };

  float acc[F8_IPC][NM][NB][4];
#pragma unroll
  for (int i = 0; i < F8_IPC; ++i)
#pragma unroll
    for (int m = 0; m < NM; ++m)
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[i][m][nb][e] = 0.f;
  float ss[NB];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) ss[nb] = 0.f;

  const int kc = K >> 8, c0 = warp * kc, c1 = c0 + kc;      // this warp's 32-k chunks
  uint4 w[F8_IPC][NM];
  float2 v[NB][4];
  load_w(c0, w);
  load_x(c0, v);
  for (int c = c0; c < c1; ++c) {
    uint4 wn[F8_IPC][NM];
    float2 vn[NB][4];
    if (c + 1 < c1) {
      load_w(c + 1, wn);
      load_x(c + 1, vn);
    }
    uint32_t bh[NB][2][2], bl[NB][2][2];                     // [n8 block][k-step][b0 | b1]
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float2 x = v[nb][q];
        if (norm) {
          ss[nb] = fmaf(x.x, x.x, ss[nb]);
          ss[nb] = fmaf(x.y, x.y, ss[nb]);
          const int k = 32 * c + 16 * (q >> 1) + 8 * (q & 1) + 2 * t;
          const __nv_bfloat162 gg = *reinterpret_cast<const __nv_bfloat162*>(p.gain + k);
          x.x *= __low2float(gg);
          x.y *= __high2float(gg);
        }
        pack_hi_lo(x.x, x.y, bh[nb][q >> 1][q & 1], bl[nb][q >> 1][q & 1]);
      }
#pragma unroll
    for (int i = 0; i < F8_IPC; ++i) {
      if (i >= n_mine) break;
#pragma unroll
      for (int m = 0; m < NM; ++m)
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          uint32_t a[4];
          f8_frag(w[i][m], s, a);
#pragma unroll
          for (int nb = 0; nb < NB; ++nb) {
            mma_bf16_16816(acc[i][m][nb], a, bh[nb][s][0], bh[nb][s][1]);
            mma_bf16_16816(acc[i][m][nb], a, bl[nb][s][0], bl[nb][s][1]);
          }
        }
    }
    if (c + 1 < c1) {
#pragma unroll
      for (int i = 0; i < F8_IPC; ++i)
#pragma unroll
        for (int m = 0; m < NM; ++m) w[i][m] = wn[i][m];
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int q = 0; q < 4; ++q) v[nb][q] = vn[nb][q];
    }
  }

  // 1 / rms of every activation row: the warps' sums of squares in warp order
  if (norm) {
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) {
      float s = ss[nb];
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      if (t == 0) ssq[warp][nb * 8 + g] = s;
    }
    __syncthreads();
    if (tid < NB * 8) {
      float s = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) s += ssq[w8][tid];
      rs[tid] = rsqrtf(s / (float)K + p.eps);
    }
  }

  // per block: the eight warps' accumulators -> shared memory, summed in warp order by the thread of each output
#pragma unroll
  for (int i = 0; i < F8_IPC; ++i) {
    if (i >= n_mine) break;
#pragma unroll
    for (int m = 0; m < NM; ++m)
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int e = 0; e < 4; ++e) red[warp][m][nb][lane * 4 + e] = acc[i][m][nb][e];
    __syncthreads();
    const int b = blockIdx.x + i * G;
    // accumulator of (block row rr, column col) in matrix m: lane 4 (rr & 7) + (col & 7) / 2, element 2 (rr >> 3) + (col & 1)
    auto sum = [&](int m, int rr, int col) {
      const int idx = (((rr & 7) << 2) + ((col & 7) >> 1)) * 4 + ((rr >> 3) << 1) + (col & 1);
      float a = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) a += red[w8][m][col >> 3][idx];
      if (norm) a *= rs[col];
      return a;
    };
    if (EPI == EPI_SWIGLU) {
      const int rr = tid & 15, e = tid >> 4;                 // w1 / w3 row 16 b + rr of batch entry e
      if (e < nu) {
        const int j = 16 * b + rr;
        const float s1 = bf16_to_f32(Ws[0][j]), s3 = bf16_to_f32(Ws[NM - 1][j]);
        gemv_epilogue<EPI>(p, st, st.slot_map[e0 + e], j, sum(0, rr, 2 * e) * s1, sum(0, rr, 2 * e + 1) * s1,
                           sum(NM - 1, rr, 2 * e) * s3, sum(NM - 1, rr, 2 * e + 1) * s3);
      }
    } else {
      const int pr = tid & 7, e = tid >> 3;                  // rows 16 b + 2 pr, + 1 of batch entry e
      const int j = 16 * b + 2 * pr;
      if (e < nu && j < M) {
        const float sa = bf16_to_f32(Ws[0][j]), sb = bf16_to_f32(Ws[0][j + 1]);
        gemv_epilogue<EPI>(p, st, st.slot_map[e0 + e], j >> 1, sum(0, 2 * pr, 2 * e) * sa, sum(0, 2 * pr, 2 * e + 1) * sa,
                           sum(0, 2 * pr + 1, 2 * e) * sb, sum(0, 2 * pr + 1, 2 * e + 1) * sb);
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------
// Widen up to five fp8 matrices (one layer's wqkv, wo, w1, w3, w2, or lm_head / speaker_cond_pos once at create) to bf16
// row-major [M, K] buffers holding q exactly, undoing the fragment-native order: the operand of the tensor-core GEMM,
// whose epilogue applies the row scales.  One thread per 16 code bytes: one 128-bit load, eight 32-bit stores.
__global__ void __launch_bounds__(256) k_f8_widen(WidenBatch m) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    if (i >= m.n) break;
    const int M = m.M[i], K = m.K[i], M16 = M & ~15;
    const size_t n_chunks = (size_t)M * K / 16, n_frag = (size_t)M16 * K / 16;
    const uint8_t* src = m.src[i];
    __nv_bfloat16* dst = m.dst[i];
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += stride) {
      const uint4 v = ldg_stream(src + c * 16);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      if (c < n_frag) {
        const size_t chunk = c >> 5;                          // 512-byte chunk: block chunk / (K / 32), k chunk % (K / 32)
        const int l = (int)(c & 31), g = l >> 2, t = l & 3;
        const size_t row = (chunk / (K >> 5)) * 16 + g;
        const int kb = (int)(chunk % (K >> 5)) * 32 + 2 * t;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int k = kb + 16 * (q >> 1) + 8 * (q & 1);
          *reinterpret_cast<uint32_t*>(dst + row * K + k) = f8x2_bf16x2(w[q] << 8);
          *reinterpret_cast<uint32_t*>(dst + (row + 8) * K + k) = f8x2_bf16x2(w[q]);
        }
      } else {                                                // row-major tail: 16 consecutive k of one row
        uint32_t o[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          o[2 * q] = f8x2_bf16x2(__byte_perm(w[q], 0u, 0x1404));
          o[2 * q + 1] = f8x2_bf16x2(__byte_perm(w[q], 0u, 0x3424));
        }
        uint4* d = reinterpret_cast<uint4*>(dst + c * 16);
        d[0] = make_uint4(o[0], o[1], o[2], o[3]);
        d[1] = make_uint4(o[4], o[5], o[6], o[7]);
      }
    }
  }
}

}  // namespace mvb
