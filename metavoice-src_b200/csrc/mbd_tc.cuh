// Tensor-core lowering of the wide multi-band-diffusion convolutions (csrc/mbd.cu): every Conv1d / ConvTranspose1d whose
// input width is a multiple of 64 channels runs as a sum of shifted GEMMs on the tensor cores,
//     out[co][n * ostride + ph] = bias[co] + emb[co] + resid[..] + sum_slot sum_ci  W_slot[co][ci] * F[n + shift_slot][col_slot + ci]
// where F is the TIME-major copy of the layer input after its GroupNorm + ReLU (k_mbd_prep_t), split into two bf16 terms
// F = hi + lo so the activations keep 16 mantissa bits, and W_slot is tap `slot` of the kernel repacked to bf16 [tap][Cout][Cin]
// at create time (k_mbd_pack_w).  Zero padding of the convolution = TMA out-of-bounds fill (negative / past-the-end rows read
// as zero), the stride-s convolution reads the same buffer through a [T/s][s * Cin] view, and the transposed convolution is
// s output phases with two taps each.  One CTA = 128 output channels x 128 time columns: A tiles (weights, 16 KB) and the
// two B tiles (hi, lo: 128 rows each) arrive by TMA into a 4-stage ring; eight consumer warps own 16 output channels each
// and run ldmatrix + mma.sync.m16n8k16 over all 128 columns, the hi and lo products accumulating into one fp32 register
// tile (tc_mainloop, shared with the weight-streaming GEMM).  The epilogue adds bias, transposes each warp's 16 x 128
// block through shared memory (the drained ring) and adds the residual / stores channel-major rows with the lanes along
// time (coalesced).
//
// Numerics: weights are rounded to bf16 (the reference's own convolutions run in TF32 under torch's cuDNN default
// `allow_tf32=True`, 10-bit mantissa on BOTH operands); activations are exact to 2^-17; accumulation is fp32.
#pragma once
#include "tc.cuh"

namespace mvb {

struct TcTaps {
  int n_slots, n_ph;
  int a_z[4][8];      // weight tap (z slice of the A map) per (phase, slot)
  int b_shift[4][8];  // row shift into the time-major activations
  int b_col[4][8];    // column base (stride-s convolution: phase * Cin)
};
struct TcConvP {
  int Cin, M, Ncols;          // K per slot; output channels per phase; GEMM columns (time rows producing outputs)
  float* out; int ldo, ostride;
  const float* bias; const float* emb; const float* resid;
  TcTaps taps;
};

constexpr int TC_STAGES = 4;
constexpr int TC_A_BYTES = 128 * 64 * 2, TC_B_BYTES = 256 * 64 * 2, TC_STAGE_BYTES = TC_A_BYTES + TC_B_BYTES;
constexpr int TC_THREADS = 288;          // TMA producer warp + 8 consumer warps
constexpr int TC_TP_LD = 128 + 4;        // epilogue transpose tile [16][TC_TP_LD] fp32 per consumer warp (inside the ring)
constexpr size_t TC_SMEM = 1024 + (size_t)TC_STAGES * TC_STAGE_BYTES + 2 * TC_STAGES * 8 + 64;
static_assert(8 * 16 * TC_TP_LD * 4 <= TC_STAGES * TC_STAGE_BYTES, "transpose tiles must fit in the ring");

static __global__ void __launch_bounds__(TC_THREADS, 1)
k_mbd_tc_conv(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBhi,
              const __grid_constant__ CUtensorMap tmBlo, const TcConvP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad_1024(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_cot = (p.M + 127) >> 7;
  const int ph = blockIdx.x / n_cot, cot = blockIdx.x - ph * n_cot;
  const int t0 = blockIdx.y * 128;
  const int nkb = p.Cin >> 6;

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&tmA);
    ptx::prefetch_tensormap(&tmBhi);
    ptx::prefetch_tensormap(&tmBlo);
  }
  // the B tile holds 128 hi rows, then the 128 lo rows
  float acc[1][16][4];
  const bool consumer = tc_mainloop<1, 16>(
      smem, TC_STAGES, TC_STAGE_BYTES, TC_A_BYTES, p.taps.n_slots * nkb, 16, 128, true,
      [&](int it, uint32_t st, uint32_t full) {
        const int slot = it / nkb, kb = it - slot * nkb;
        const int row = t0 + p.taps.b_shift[ph][slot], col = p.taps.b_col[ph][slot] + kb * 64;
        ptx::tma_load_3d(st, &tmA, full, kb * 64, cot * 128, p.taps.a_z[ph][slot]);
        ptx::tma_load_2d(st + TC_A_BYTES, &tmBhi, full, col, row);
        ptx::tma_load_2d(st + TC_A_BYTES + TC_B_BYTES / 2, &tmBlo, full, col, row);
      },
      acc);
  if (!consumer) return;

  // consumers: warp w owns output channels [16 (w - 1), 16 w) of the tile
  const int w16 = 16 * (warp - 1);
  // Epilogue: accumulator (lane holds channels w16 + lane/4 (+8), columns 8c + 2(lane%4) (+1)) -> padded smem tile in the
  // drained ring -> global with lane = TIME, so that the residual reads and the stores are contiguous 128-byte rows
  // instead of scattered sectors (the channel-major activations have stride ldo between channels).
  asm volatile("bar.sync 1, 256;" ::: "memory");   // every consumer is done with the ring
  float* tp = reinterpret_cast<float*>(smem) + (warp - 1) * (16 * TC_TP_LD);
  const int co_w = cot * 128 + w16;               // first channel of this warp
  if (co_w < p.M) {
    const int rows = min(16, p.M - co_w);
#pragma unroll
    for (int h8 = 0; h8 < 2; ++h8) {
      const int r = (lane >> 2) + 8 * h8, co = co_w + r;
      const float add = co < p.M ? (p.bias ? p.bias[co] : 0.f) + (p.emb ? p.emb[co] : 0.f) : 0.f;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        tp[r * TC_TP_LD + 8 * c + 2 * (lane & 3)] = acc[0][c][2 * h8] + add;
        tp[r * TC_TP_LD + 8 * c + 2 * (lane & 3) + 1] = acc[0][c][2 * h8 + 1] + add;
      }
    }
    __syncwarp();
    for (int c0 = 0; c0 < 128 && t0 + c0 < p.Ncols; c0 += 32) {
      const int n = t0 + c0 + lane;
      if (n < p.Ncols) {
        const size_t col = (size_t)n * p.ostride + ph;
        // residual reads in batches of 8 rows: issued back to back, not one dependent load -> store pair per row
        for (int r0 = 0; r0 < rows; r0 += 8) {
          float rv[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int r = min(r0 + j, rows - 1);
            rv[j] = p.resid ? __ldg(p.resid + (size_t)(co_w + r) * p.ldo + col) : 0.f;
          }
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (r0 + j < rows) p.out[(size_t)(co_w + r0 + j) * p.ldo + col] = tp[(r0 + j) * TC_TP_LD + c0 + lane] + rv[j];
        }
      }
    }
  }
}

// Time-major two-term bf16 copy of a layer input: hi/lo[t][c] = split(f(x[c][t])), f = relu(GroupNorm) when stats != null;
// rows T .. Tpad-1 are written as zero (right padding of the strided convolution).  Tile: 64 channels x 32 samples.
static __global__ void __launch_bounds__(256) k_mbd_prep_t(const float* __restrict__ x, int C, int Cp, int T, int Tpad, const float* __restrict__ stats,
                                                           const float* __restrict__ gw, const float* __restrict__ gb, int cpg,
                                                           __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  __shared__ float tile[64][33];
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 64;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = c0 + ty * 8 + i, t = t0 + tx;
    float v = 0.f;
    if (c < C && t < T) {
      v = x[(size_t)c * T + t];
      if (stats) {
        const int g = c / cpg;
        v = fmaxf((v - stats[2 * g]) * stats[2 * g + 1] * gw[c] + gb[c], 0.f);
      }
    }
    tile[ty * 8 + i][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int tl = ty * 4 + i, t = t0 + tl, c = c0 + 2 * tx;
    if (t < Tpad && c < Cp) {       // columns C .. Cp-1 (channel padding to a multiple of 64) are written as zero
      uint32_t h2, l2;
      pack_hi_lo(tile[2 * tx][tl], tile[2 * tx + 1][tl], h2, l2);
      *reinterpret_cast<uint32_t*>(hi + (size_t)t * Cp + c) = h2;
      *reinterpret_cast<uint32_t*>(lo + (size_t)t * Cp + c) = l2;
    }
  }
}

// Weight repack to bf16 [tap][Cout][Cp]: transposed = 0: w is Conv1d [Cout][Cin][K]; 1: ConvTranspose1d [Cin][Cout][K].
// (Cp = Cin rounded up to a multiple of 64; the padding columns are zero.)
static __global__ void k_mbd_pack_w(const float* __restrict__ w, int Cout, int Cin, int Cp, int K, int transposed, __nv_bfloat16* __restrict__ out) {
  const size_t n = (size_t)K * Cout * Cp;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int ci = (int)(i % Cp), co = (int)((i / Cp) % Cout), k = (int)(i / ((size_t)Cp * Cout));
    const size_t src = transposed ? ((size_t)ci * Cout + co) * K + k : ((size_t)co * Cin + ci) * K + k;
    out[i] = __float2bfloat16_rn(ci < Cin ? w[src] : 0.f);
  }
}

}  // namespace mvb
