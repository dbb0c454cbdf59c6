// EnCodec-24 kHz decode path of the vocoder (SURVEY.md row a17, first half): RVQ decode -> SEANet decoder.
// This is what `mbd.tokens_to_wav` (fam/llm/decoders.py:85 -> audiocraft 1.2.0) computes first, as the loudness /
// band-energy reference and as the diffusion condition (`decode_latent`).  audiocraft delegates the 24 kHz codec to
// transformers.EncodecModel; operator semantics follow modeling_encodec.py (cited per kernel).  fp32 throughout
// (the reference forces fp32 autocast for the vocoder, decoders.py:84).
//
// Activations are [C][T] fp32 per utterance (time contiguous): every conv streams its input window through a
// shared-memory line buffer (128-bit coalesced loads of the tile body, scalar loads for the K-1 halo samples), keeps an
// 8-channel x 4-sample register tile per thread and writes it back with 128-bit stores.
#include <cuda_runtime.h>

#include <vector>

#include "common.cuh"
#include "host.cuh"

using namespace mvb;

namespace {

__device__ __forceinline__ float elu1(float v) { return v > 0.f ? v : expm1f(v); }

// latent[c][t] = sum_q codebook_q[codes[q][t]][c]     (EncodecResidualVectorQuantizer.decode)
// One tile of 32 frames from t0: codes [n_q, T] -> out [dim, T].
__device__ __forceinline__ void rvq_tile(const int* __restrict__ codes, int n_q, int T, const float* const* __restrict__ books,
                                         int dim, float* __restrict__ out, int t0) {
  __shared__ float tile[32][129];
  const int c = threadIdx.x;
  for (int i = 0; i < 32; ++i) {
    const int t = t0 + i;
    float acc = 0.f;
    if (t < T && c < dim)
      for (int q = 0; q < n_q; ++q) acc += books[q][(size_t)codes[(size_t)q * T + t] * dim + c];
    tile[i][c] = acc;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 32 * dim; idx += 128) {
    const int cc = idx / 32, i = idx - cc * 32;
    if (t0 + i < T) out[(size_t)cc * T + t0 + i] = tile[i][cc];
  }
}

__global__ void __launch_bounds__(128) k_rvq_decode(const int* __restrict__ codes, int n_q, int T, const float* const* __restrict__ books,
                                                    int dim, float* __restrict__ out) {
  const int b = blockIdx.y;
  rvq_tile(codes + (size_t)b * n_q * T, n_q, T, books, dim, out + (size_t)b * dim * T, blockIdx.x * 32);
}

// Causal Conv1d, stride 1, dilation 1, reflect padding of K-1 samples on the left (EncodecConv1d, causal branch),
// optional ELU on the input (the nn.ELU() that precedes the conv in the stack) and optional accumulation into y
// (residual / shortcut sum of EncodecResnetBlock).  Tile: 32 output channels x 256 samples, 16 input channels per pass.
// One tile of one sequence: xb [Cin, T] -> yb [Cout, T], samples t0 .. t0 + 255, output channels co0 .. co0 + 31.
template <int K>
__device__ __forceinline__ void conv1d_tile(const float* __restrict__ xb, int Cin, int T, const float* __restrict__ w,
                                            const float* __restrict__ bias, float* __restrict__ yb, int Cout, int elu_in,
                                            int accumulate, int t0, int co0) {
  constexpr int CI = 16, TT = 256, CO = 32;
  __shared__ float xs[CI][TT + K - 1 + 1];
  __shared__ float ws[CO][CI][K];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;    // 64 time groups of 4 samples x 4 groups of 8 channels
  // 128-bit loads and stores need T % 4 == 0 and 16-byte aligned sequence bases (a batched segment may start anywhere)
  const bool vec = (T & 3) == 0 && ((reinterpret_cast<uintptr_t>(xb) | reinterpret_cast<uintptr_t>(yb)) & 15) == 0;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int c0 = 0; c0 < Cin; c0 += CI) {
    __syncthreads();
    // line buffer: samples t0-(K-1) .. t0+TT-1 of 16 channels.  The TT-sample body is streamed with 128-bit loads
    // (rows are 16-byte aligned when T % 4 == 0, which holds for every layer of the decoder: T = frames x 8 x ...);
    // the K-1 halo samples in front are loaded one by one, negative times reflect (x[-j] = x[j]).
    if (vec) {
      for (int i = threadIdx.x; i < CI * (TT / 4); i += 256) {
        const int ci = i / (TT / 4), q4 = i - ci * (TT / 4);
        const int t = t0 + 4 * q4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c0 + ci < Cin && t < T) {          // T % 4 == 0: a float4 is either fully inside or fully outside
          v = *reinterpret_cast<const float4*>(xb + (size_t)(c0 + ci) * T + t);
          if (elu_in) { v.x = elu1(v.x); v.y = elu1(v.y); v.z = elu1(v.z); v.w = elu1(v.w); }
        }
        float* d = &xs[ci][K - 1 + 4 * q4];
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
      }
    }
    for (int i = threadIdx.x; i < CI * (vec ? K - 1 : TT + K - 1); i += 256) {
      const int span = vec ? K - 1 : TT + K - 1;
      const int ci = i / span, tt = i - ci * span;
      int t = t0 + tt - (K - 1);
      if (t < 0) t = -t;
      float v = 0.f;
      if (c0 + ci < Cin && t < T) {
        v = xb[(size_t)(c0 + ci) * T + t];
        if (elu_in) v = elu1(v);
      }
      xs[ci][tt] = v;
    }
    for (int i = threadIdx.x; i < CO * CI * K; i += 256) {
      const int co = i / (CI * K), r = i - co * (CI * K), ci = r / K, k = r - ci * K;
      ws[co][ci][k] = (co0 + co < Cout && c0 + ci < Cin) ? w[((size_t)(co0 + co) * Cin + c0 + ci) * K + k] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int ci = 0; ci < CI; ++ci) {
      float xv[4 + K - 1];
#pragma unroll
      for (int j = 0; j < 4 + K - 1; ++j) xv[j] = xs[ci][tx * 4 + j];
#pragma unroll
      for (int k = 0; k < K; ++k)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float wv = ws[ty * 8 + i][ci][k];
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(wv, xv[j + k], acc[i][j]);
        }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int co = co0 + ty * 8 + i;
    if (co >= Cout) continue;
    const float bv = bias ? bias[co] : 0.f;
    const int tb = t0 + tx * 4;
    if (vec && tb < T) {                       // 128-bit coalesced store of the thread's 4 consecutive samples
      float4* o = reinterpret_cast<float4*>(yb + (size_t)co * T + tb);
      float4 v = make_float4(acc[i][0] + bv, acc[i][1] + bv, acc[i][2] + bv, acc[i][3] + bv);
      if (accumulate) { const float4 p = *o; v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w; }
      *o = v;
      continue;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int t = t0 + tx * 4 + j;
      if (t < T) {
        float* o = yb + (size_t)co * T + t;
        const float v = acc[i][j] + bv;
        *o = accumulate ? *o + v : v;
      }
    }
  }
}

template <int K>
__global__ void __launch_bounds__(256) k_conv1d(const float* __restrict__ x, int Cin, int T, const float* __restrict__ w,
                                                const float* __restrict__ bias, float* __restrict__ y, int Cout, int elu_in, int accumulate) {
  const int b = blockIdx.z;
  conv1d_tile<K>(x + (size_t)b * Cin * T, Cin, T, w, bias, y + (size_t)b * Cout * T, Cout, elu_in, accumulate, blockIdx.x * 256,
                 blockIdx.y * 32);
}

// ConvTranspose1d(k = 2r, stride r) trimmed by r samples on the right (EncodecConvTranspose1d, causal) with the
// preceding ELU fused:  y[co][t*r + p] = b[co] + sum_ci w[ci][co][p] * e[ci][t] + w[ci][co][p + r] * e[ci][t-1].
// One tile of one sequence: xb [Cin, T] -> yb [Cout, T r], input frames t0 .. t0 + 31; sm = the dynamic shared memory.
__device__ __forceinline__ void convtr1d_tile(const float* __restrict__ xb, int Cin, int T, const float* __restrict__ w,
                                              const float* __restrict__ bias, float* __restrict__ yb, int Cout, int r, int t0,
                                              int co0, float* sm) {
  constexpr int CI = 16, TI = 32, CO = 32;
  float* xs = sm;                       // [CI][TI + 1]   (index 0 = t0 - 1)
  float* ws = sm + CI * (TI + 1);       // [CI][CO][2r]
  const int ox = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int n_out = TI * r;             // outputs of this tile
  float acc[8][4];
  int tl[4], pp[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int o = ox + 64 * j;
    tl[j] = o / r;
    pp[j] = o - tl[j] * r;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int c0 = 0; c0 < Cin; c0 += CI) {
    __syncthreads();
    for (int i = threadIdx.x; i < CI * (TI + 1); i += 256) {
      const int ci = i / (TI + 1), tt = i - ci * (TI + 1);
      const int t = t0 + tt - 1;
      float v = 0.f;
      if (c0 + ci < Cin && t >= 0 && t < T) v = elu1(xb[(size_t)(c0 + ci) * T + t]);
      xs[i] = v;
    }
    for (int i = threadIdx.x; i < CI * CO * 2 * r; i += 256) {
      const int ci = i / (CO * 2 * r), rem = i - ci * (CO * 2 * r), co = rem / (2 * r), k = rem - co * (2 * r);
      ws[i] = (c0 + ci < Cin && co0 + co < Cout) ? w[((size_t)(c0 + ci) * Cout + co0 + co) * (2 * r) + k] : 0.f;
    }
    __syncthreads();
    for (int ci = 0; ci < CI; ++ci) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (ox + 64 * j < n_out) {
          const float e1 = xs[ci * (TI + 1) + tl[j] + 1], e0 = xs[ci * (TI + 1) + tl[j]];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float* wp = ws + ((size_t)ci * CO + ty * 8 + i) * 2 * r;
            acc[i][j] = fmaf(wp[pp[j]], e1, fmaf(wp[pp[j] + r], e0, acc[i][j]));
          }
        }
      }
    }
  }
  const int To = T * r;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int co = co0 + ty * 8 + i;
    if (co >= Cout) continue;
    const float bv = bias[co];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = ox + 64 * j;
      const int n = t0 * r + o;
      if (o < n_out && n < To) yb[(size_t)co * To + n] = acc[i][j] + bv;
    }
  }
}

__global__ void __launch_bounds__(256) k_convtr1d(const float* __restrict__ x, int Cin, int T, const float* __restrict__ w,
                                                  const float* __restrict__ bias, float* __restrict__ y, int Cout, int r) {
  extern __shared__ float sm[];
  const int b = blockIdx.z;
  convtr1d_tile(x + (size_t)b * Cin * T, Cin, T, w, bias, y + (size_t)b * Cout * T * r, Cout, r, blockIdx.x * 32, blockIdx.y * 32, sm);
}

// One LSTM layer (EncodecLSTM: nn.LSTM, gate order i, f, g, o, zero initial state), persistent over time:
// CTA c owns hidden units [4c, 4c+4) = 16 gate rows of W_hh held in shared memory; h_{t-1} is exchanged through
// global memory and one grid-wide arrive/wait per step.  pre[row][t] = W_ih x_t + b_ih + b_hh is computed beforehand
// by k_conv1d<1>.  The skip connection of EncodecLSTM (output + input) is fused into the last layer's store.
__global__ void __launch_bounds__(128) k_lstm_layer(const float* __restrict__ pre, const float* __restrict__ whh, int H, int T,
                                                    float* __restrict__ hbuf /*[2][H]*/, unsigned* bar, float* __restrict__ out,
                                                    const float* __restrict__ skip) {
  extern __shared__ float sm[];
  float* wsm = sm;               // [16][H]
  float* hs = sm + 16 * H;       // [H]
  __shared__ float gates[16];
  const int cta = blockIdx.x, tid = threadIdx.x;
  const int u0 = cta * 4;
  for (int i = tid; i < 16 * H; i += 128) {
    const int r = i / H, k = i - r * H;
    const int grow = (r >> 2) * H + u0 + (r & 3);
    wsm[i] = whh[(size_t)grow * H + k];
  }
  float c_state = 0.f;
  const int row = tid >> 3, part = tid & 7;      // 16 rows x 8 lanes
  const int seg = H / 8;
  __syncthreads();
  for (int t = 0; t < T; ++t) {
    if (t > 0) {
      if (tid == 0) wait_counter(bar, (unsigned)t * gridDim.x);
      __syncthreads();
      const float* hp = hbuf + (size_t)((t - 1) & 1) * H;
      for (int k = tid; k < H; k += 128) hs[k] = __ldcg(hp + k);
    } else {
      for (int k = tid; k < H; k += 128) hs[k] = 0.f;
    }
    __syncthreads();
    float a = 0.f;
    const float* wr = wsm + row * H + part * seg;
    const float* hh = hs + part * seg;
#pragma unroll 8
    for (int k = 0; k < seg; ++k) a = fmaf(wr[k], hh[k], a);
    a += __shfl_xor_sync(0xffffffffu, a, 4);
    a += __shfl_xor_sync(0xffffffffu, a, 2);
    a += __shfl_xor_sync(0xffffffffu, a, 1);
    if (part == 0) {
      const int grow = (row >> 2) * H + u0 + (row & 3);
      gates[row] = a + pre[(size_t)grow * T + t];
    }
    __syncthreads();
    if (tid < 4) {
      const float ig = 1.f / (1.f + expf(-gates[tid]));
      const float fg = 1.f / (1.f + expf(-gates[4 + tid]));
      const float gg = tanhf(gates[8 + tid]);
      const float og = 1.f / (1.f + expf(-gates[12 + tid]));
      c_state = fg * c_state + ig * gg;
      const float h = og * tanhf(c_state);
      hbuf[(size_t)(t & 1) * H + u0 + tid] = h;
      out[(size_t)(u0 + tid) * T + t] = skip ? h + skip[(size_t)(u0 + tid) * T + t] : h;
    }
    __syncthreads();
    if (tid == 0) red_release_inc(bar);
  }
}

// ---- batched decode: B utterances of T_i frames in one launch set ------------------------------------------------------
// Every activation is concatenated per utterance: a layer with C channels at m samples per frame holds utterance i as a
// [C, T_i m] block starting at element C off_i m (off_i = T_0 + ... + T_{i-1}).  blockIdx.z is the utterance; tiles past
// its end return, so every tile computes exactly what the same tile of the single-utterance launch computes.
constexpr int VOC_MAX_BATCH = 32;
struct Seg { int T, off; };

__global__ void __launch_bounds__(128) k_rvq_decode_b(const int* __restrict__ codes, int n_q, const Seg* __restrict__ segs,
                                                      const float* const* __restrict__ books, int dim, float* __restrict__ out) {
  const Seg g = segs[blockIdx.z];
  const int t0 = blockIdx.x * 32;
  if (t0 >= g.T) return;
  rvq_tile(codes + (size_t)n_q * g.off, n_q, g.T, books, dim, out + (size_t)dim * g.off, t0);
}

template <int K>
__global__ void __launch_bounds__(256) k_conv1d_b(const float* __restrict__ x, int Cin, const Seg* __restrict__ segs, int m,
                                                  const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ y,
                                                  int Cout, int elu_in, int accumulate) {
  const Seg g = segs[blockIdx.z];
  const int T = g.T * m, t0 = blockIdx.x * 256;
  if (t0 >= T) return;
  const size_t off = (size_t)g.off * m;
  conv1d_tile<K>(x + off * Cin, Cin, T, w, bias, y + off * Cout, Cout, elu_in, accumulate, t0, blockIdx.y * 32);
}

// input at m samples per frame, output at m r
__global__ void __launch_bounds__(256) k_convtr1d_b(const float* __restrict__ x, int Cin, const Seg* __restrict__ segs, int m,
                                                    const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ y,
                                                    int Cout, int r) {
  extern __shared__ float sm[];
  const Seg g = segs[blockIdx.z];
  const int T = g.T * m, t0 = blockIdx.x * 32;
  if (t0 >= T) return;
  const size_t off = (size_t)g.off * m;
  convtr1d_tile(x + off * Cin, Cin, T, w, bias, y + off * r * Cout, Cout, r, t0, blockIdx.y * 32, sm);
}

// k_lstm_layer for n <= 32 sequences at once: one grid barrier per step of the longest sequence instead of one per step of
// every sequence.  CTA c still owns hidden units [4c, 4c+4) and holds their 16 W_hh rows in shared memory, loaded once;
// each step it computes those 16 gate rows for every sequence still running (t < T_i) and the finished ones stop writing.
// Every pre-activation is summed exactly as k_lstm_layer sums it (8 lanes x H/8 consecutive products, then xor-shuffles
// 4 / 2 / 1), so each sequence is bit-identical to its single-sequence run.  Shared memory rows are padded by one float
// per H/8 segment: the 8 lanes of a row and the 4 rows of a warp then read 32 different banks.
// pre: per sequence [4H, T_i] at 4H off_i; out / skip: [H, T_i] at H off_i; hbuf [2][n][H].
__host__ __device__ constexpr int lstm_b_ld(int H) { return H + 8; }

__global__ void __launch_bounds__(128) k_lstm_layer_b(const float* __restrict__ pre, const float* __restrict__ whh, int H,
                                                      const Seg* __restrict__ segs, int n, int T_max, float* __restrict__ hbuf,
                                                      unsigned* bar, float* __restrict__ out, const float* __restrict__ skip) {
  extern __shared__ float sm[];
  const int seg = H / 8, ld = lstm_b_ld(H);
  float* wsm = sm;                 // [16][ld]
  float* hs = sm + 16 * ld;        // [round_up(n, 4)][ld]
  __shared__ float gates[VOC_MAX_BATCH][16];
  __shared__ int Ts[VOC_MAX_BATCH], offs[VOC_MAX_BATCH];
  const int cta = blockIdx.x, tid = threadIdx.x;
  const int u0 = cta * 4;
  const int n4 = (n + 3) & ~3;
  auto at = [seg](int k) { const int p = k / seg; return p * (seg + 1) + (k - p * seg); };   // padded column of k
  for (int i = tid; i < 16 * H; i += 128) {
    const int r = i / H, k = i - r * H;
    const int grow = (r >> 2) * H + u0 + (r & 3);
    wsm[r * ld + at(k)] = whh[(size_t)grow * H + k];
  }
  if (tid < n) { Ts[tid] = segs[tid].T; offs[tid] = segs[tid].off; }
  float c_state = 0.f;
  const int row = tid >> 3, part = tid & 7;      // 16 rows x 8 lanes
  const int cb = tid >> 2, cu = tid & 3;         // cell update: sequence cb, unit u0 + cu
  __syncthreads();
  for (int t = 0; t < T_max; ++t) {
    if (t > 0) {
      if (tid == 0) wait_counter(bar, (unsigned)t * gridDim.x);
      __syncthreads();
      for (int b = 0; b < n; ++b) {
        if (t >= Ts[b]) continue;
        const float* hp = hbuf + ((size_t)((t - 1) & 1) * n + b) * H;
        for (int k = tid; k < H; k += 128) hs[b * ld + at(k)] = __ldcg(hp + k);
      }
    } else {
      for (int k = tid; k < n4 * ld; k += 128) hs[k] = 0.f;
    }
    __syncthreads();
    const float* wr = wsm + row * ld + part * (seg + 1);
    for (int b0 = 0; b0 < n; b0 += 4) {
      // four sequences share each W_hh load; every accumulator is its own sequential fmaf chain
      float a[4] = {0.f, 0.f, 0.f, 0.f};
      const float* hh = hs + b0 * ld + part * (seg + 1);
#pragma unroll 4
      for (int k = 0; k < seg; ++k) {
        const float wv = wr[k];
#pragma unroll
        for (int j = 0; j < 4; ++j) a[j] = fmaf(wv, hh[j * ld + k], a[j]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        a[j] += __shfl_xor_sync(0xffffffffu, a[j], 4);
        a[j] += __shfl_xor_sync(0xffffffffu, a[j], 2);
        a[j] += __shfl_xor_sync(0xffffffffu, a[j], 1);
        const int b = b0 + j;
        if (part == 0 && b < n && t < Ts[b]) {
          const int grow = (row >> 2) * H + u0 + (row & 3);
          gates[b][row] = a[j] + pre[(size_t)offs[b] * 4 * H + (size_t)grow * Ts[b] + t];
        }
      }
    }
    __syncthreads();
    if (cb < n && t < Ts[cb]) {
      const float* gt = gates[cb];
      const float ig = 1.f / (1.f + expf(-gt[cu]));
      const float fg = 1.f / (1.f + expf(-gt[4 + cu]));
      const float gg = tanhf(gt[8 + cu]);
      const float og = 1.f / (1.f + expf(-gt[12 + cu]));
      c_state = fg * c_state + ig * gg;
      const float h = og * tanhf(c_state);
      hbuf[((size_t)(t & 1) * n + cb) * H + u0 + cu] = h;
      const size_t o = (size_t)offs[cb] * H + (size_t)(u0 + cu) * Ts[cb] + t;
      out[o] = skip ? h + skip[o] : h;
    }
    __syncthreads();
    if (tid == 0) red_release_inc(bar);
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
struct mvb_voc {
  mvb_voc_config cfg;
  const char* arena;
  std::vector<uint64_t> off;
  char* ws;
  float *bufA, *bufB, *bufC, *pre;
  float* hbuf;
  unsigned* bar;
  const float** books_dev;
  const float* w(int i) const { return reinterpret_cast<const float*>(arena + off[i]); }
};

// tensor order in the arena (fp32, weight norm folded by the loader):
//   codebooks[n_q] | conv_in {w,b} | lstm l0 {w_ih, w_hh, b_ih+b_hh} | lstm l1 {...} |
//   per ratio: up {w,b}, res.c1 {w,b}, res.c2 {w,b}, res.shortcut {w,b} | conv_out {w,b}
static int voc_n_tensors(const mvb_voc_config* c) { return c->n_q + 2 + 6 + c->n_ratios * 8 + 2; }

struct VocLayout { size_t A, B, C, pre, h, bar, books, total; };

// Elements of the largest decoder activation over T frames (channels x samples, over the upsampling stages).
static size_t voc_max_elems(const mvb_voc_config* c, size_t T) {
  int ch = c->n_filters << c->n_ratios;   // 512
  size_t maxelems = (size_t)ch * T, Tl = T;
  for (int i = 0; i < c->n_ratios; ++i) {
    Tl *= c->ratios[i];
    ch >>= 1;
    if ((size_t)ch * Tl > maxelems) maxelems = (size_t)ch * Tl;
  }
  return maxelems;
}

static VocLayout voc_layout(const mvb_voc_config* c) {
  const size_t T = c->max_frames;
  const size_t maxelems = voc_max_elems(c, T);
  const size_t top = (size_t)(c->n_filters << c->n_ratios);
  VocLayout L;
  WsBump ws;
  L.A = ws.take(maxelems * 4); L.B = ws.take(maxelems * 4); L.C = ws.take(maxelems * 4);
  L.pre = ws.take(4 * top * T * 4);
  L.h = ws.take(2 * top * 4);
  L.bar = ws.take(256);
  L.books = ws.take(64 * sizeof(void*));
  L.total = ws.end;
  return L;
}

// k_lstm_layer: W_hh slice [16][H] + h [H] of dynamic shared memory per CTA, under the 100 KB opt-in set below
constexpr int LSTM_SMEM_LIMIT = 100 * 1024;
static size_t lstm_smem(int H) { return (size_t)(16 * H + H) * 4; }

static int lstm_set_smem_limit() {
  static PerDeviceOnce attr;
  if (attr.pending()) {
    MVB_CK(cudaFuncSetAttribute(k_lstm_layer, cudaFuncAttributeMaxDynamicSharedMemorySize, LSTM_SMEM_LIMIT));
    attr.mark();
  }
  return MVB_OK;
}

// k_lstm_layer_b: W_hh slice + h of round_up(n, 4) sequences, rows padded to lstm_b_ld(H)
static size_t lstm_b_smem(int H, int n) { return (size_t)(16 + ((n + 3) & ~3)) * lstm_b_ld(H) * 4; }

static int lstm_b_set_smem_limit() {
  static PerDeviceOnce attr;
  if (attr.pending()) {
    MVB_CK(cudaFuncSetAttribute(k_lstm_layer_b, cudaFuncAttributeMaxDynamicSharedMemorySize, LSTM_SMEM_LIMIT));
    attr.mark();
  }
  return MVB_OK;
}

// The H / 4 CTAs of one LSTM layer meet at a grid-wide barrier every step, so all of them must be resident at once on
// the current device; a layer that cannot be is rejected instead of launched (it would wait forever).
template <class Kernel>
static int check_coresident(Kernel kernel, int H, size_t smem) {
  int dev = 0, n_sm = 0, per_sm = 0;
  if (int e = current_device(&dev, &n_sm)) return e;
  MVB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 128, smem));
  if (H / 4 > per_sm * n_sm)
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "LSTM width %d: %d CTAs cannot be co-resident (%d per SM x %d SMs)", H, H / 4,
                          per_sm, n_sm);
  return MVB_OK;
}

static int lstm_check_coresident(int H) {
  if (int e = lstm_set_smem_limit()) return e;
  return check_coresident(k_lstm_layer, H, lstm_smem(H));
}

static int lstm_b_check_coresident(int H, int n) {
  if (int e = lstm_b_set_smem_limit()) return e;
  return check_coresident(k_lstm_layer_b, H, lstm_b_smem(H, n));
}

static int voc_validate(const mvb_voc_config* c) {
  if (!c) return mvb::set_error(MVB_ERR_ARG, "null config");
  if (c->n_ratios < 1 || c->n_ratios > 8 || c->n_q < 1 || c->n_q > 32) return mvb::set_error(MVB_ERR_ARG, "bad codec shape");
  if (c->hidden > 128) return mvb::set_error(MVB_ERR_UNSUPPORTED, "codebook dim > 128");
  const int top = c->n_filters << c->n_ratios;
  if (top < 32 || top % 32 || lstm_smem(top) > (size_t)LSTM_SMEM_LIMIT)
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "LSTM width %d unsupported", top);
  for (int i = 0; i < c->n_ratios; ++i)
    if (c->ratios[i] < 1 || c->ratios[i] > 8) return mvb::set_error(MVB_ERR_UNSUPPORTED, "upsampling ratio out of range");
  if (c->kernel != 7 || c->res_kernel != 3 || c->last_kernel != 7) return mvb::set_error(MVB_ERR_UNSUPPORTED, "kernel sizes must be 7/3/7");
  if (c->max_frames < 8) return mvb::set_error(MVB_ERR_ARG, "max_frames too small");
  return MVB_OK;
}

extern "C" size_t mvb_voc_workspace_bytes(const mvb_voc_config* c) {
  if (voc_validate(c)) return 0;
  return voc_layout(c).total;
}

extern "C" int mvb_voc_create(const mvb_voc_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets, void* d_ws,
                              mvb_voc** out) {
  if (int e = voc_validate(cfg)) return e;
  if (!d_arena || !offsets || !d_ws || !out) return mvb::set_error(MVB_ERR_ARG, "null pointer argument");
  if (int e = check_offsets(offsets, voc_n_tensors(cfg), arena_bytes, "vocoder: weight offset")) return e;
  if (int e = lstm_check_coresident(cfg->n_filters << cfg->n_ratios)) return e;
  Building<mvb_voc> hb(new mvb_voc(), mvb_voc_destroy);
  mvb_voc* h = hb.get();
  h->cfg = *cfg;
  h->arena = reinterpret_cast<const char*>(d_arena);
  h->off.assign(offsets, offsets + voc_n_tensors(cfg));
  h->ws = reinterpret_cast<char*>(d_ws);
  const VocLayout L = voc_layout(cfg);
  h->bufA = (float*)(h->ws + L.A); h->bufB = (float*)(h->ws + L.B); h->bufC = (float*)(h->ws + L.C); h->pre = (float*)(h->ws + L.pre);
  h->hbuf = (float*)(h->ws + L.h); h->bar = (unsigned*)(h->ws + L.bar); h->books_dev = (const float**)(h->ws + L.books);
  std::vector<const float*> books(cfg->n_q);
  for (int q = 0; q < cfg->n_q; ++q) books[q] = h->w(q);
  MVB_CK(cudaMemcpy(h->books_dev, books.data(), sizeof(void*) * cfg->n_q, cudaMemcpyHostToDevice));
  *out = hb.release();
  return MVB_OK;
}

extern "C" int mvb_voc_destroy(mvb_voc* h) {
  delete h;
  return MVB_OK;
}

template <int K>
static cudaError_t conv(cudaStream_t s, const float* x, int Cin, int T, const float* w, const float* b, float* y, int Cout, int elu, int acc) {
  dim3 grid((T + 255) / 256, (Cout + 31) / 32, 1);
  k_conv1d<K><<<grid, 256, 0, s>>>(x, Cin, T, w, b, y, Cout, elu, acc);
  return cudaGetLastError();
}

static cudaError_t convtr(cudaStream_t s, const float* x, int Cin, int T, const float* w, const float* b, float* y, int Cout, int r) {
  const size_t smem = (size_t)(16 * 33 + 16 * 32 * 2 * r) * 4;
  k_convtr1d<<<dim3((T + 31) / 32, (Cout + 31) / 32, 1), 256, smem, s>>>(x, Cin, T, w, b, y, Cout, r);
  return cudaGetLastError();
}

// One LSTM layer over pre [4H, T]; the caller has checked lstm_check_coresident(H) and set the shared-memory limit.
static cudaError_t lstm(cudaStream_t s, const float* pre, const float* whh, int H, int T, float* hbuf, unsigned* bar, float* out,
                        const float* skip) {
  cudaError_t e = cudaMemsetAsync(bar, 0, 4, s);
  if (e != cudaSuccess) return e;
  k_lstm_layer<<<H / 4, 128, lstm_smem(H), s>>>(pre, whh, H, T, hbuf, bar, out, skip);
  return cudaGetLastError();
}

// RVQ decode only: the diffusion condition `decode_latent` (and the decoder's input).  d_codes int32 [n_q, T].
extern "C" int mvb_voc_decode_latent(mvb_voc* h, const int32_t* d_codes, int32_t T, float* d_latent, void* stream) {
  if (!h || !d_codes || !d_latent) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (T < 1 || T > h->cfg.max_frames) return mvb::set_error(MVB_ERR_ARG, "frame count %d out of range", T);
  k_rvq_decode<<<dim3((T + 31) / 32, 1), 128, 0, (cudaStream_t)stream>>>(d_codes, h->cfg.n_q, T, h->books_dev, h->cfg.hidden, d_latent);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

// codes int32 [n_q, T] -> waveform fp32 [T * prod(ratios)]   (== EncodecModel.decode for one chunk)
extern "C" int mvb_voc_decode(mvb_voc* h, const int32_t* d_codes, int32_t T, float* d_wav, void* stream) {
  if (!h || !d_codes || !d_wav) return mvb::set_error(MVB_ERR_ARG, "null argument");
  const mvb_voc_config& c = h->cfg;
  if (T < 8 || T > c.max_frames) return mvb::set_error(MVB_ERR_ARG, "frame count %d out of range [8, %d]", T, c.max_frames);
  cudaStream_t s = (cudaStream_t)stream;
  const int top = c.n_filters << c.n_ratios;
  int ti = c.n_q;
  float *A = h->bufA, *B = h->bufB, *Cc = h->bufC;
  if (int e = mvb_voc_decode_latent(h, d_codes, T, A, stream)) return e;
  MVB_CK(conv<7>(s, A, c.hidden, T, h->w(ti), h->w(ti + 1), B, top, 0, 0));      // conv_in
  ti += 2;
  // LSTM: x = B;  layer 0 -> A ; layer 1 (+ skip x) -> Cc
  if (int e = lstm_set_smem_limit()) return e;
  const float* lin = B;
  float* louts[2] = {A, Cc};
  for (int l = 0; l < 2; ++l) {
    MVB_CK(conv<1>(s, lin, top, T, h->w(ti), h->w(ti + 2), h->pre, 4 * top, 0, 0));   // W_ih x + (b_ih + b_hh)
    MVB_CK(lstm(s, h->pre, h->w(ti + 1), top, T, h->hbuf, h->bar, louts[l], l == 1 ? B : nullptr));
    lin = louts[l];
    ti += 3;
  }
  float* x = Cc;           // current activation
  float* f1 = A;
  float* f2 = B;
  int ch = top, Tl = T;
  for (int i = 0; i < c.n_ratios; ++i) {
    const int r = c.ratios[i], co = ch / 2;
    MVB_CK(convtr(s, x, ch, Tl, h->w(ti), h->w(ti + 1), f1, co, r));
    Tl *= r; ch = co;
    // resnet block: y = shortcut(u) + conv_k1(elu(conv_k3(elu(u))))
    MVB_CK(conv<3>(s, f1, ch, Tl, h->w(ti + 2), h->w(ti + 3), f2, ch / c.compress, 1, 0));
    MVB_CK(conv<1>(s, f1, ch, Tl, h->w(ti + 6), h->w(ti + 7), x, ch, 0, 0));
    MVB_CK(conv<1>(s, f2, ch / c.compress, Tl, h->w(ti + 4), h->w(ti + 5), x, ch, 1, 1));
    ti += 8;
  }
  MVB_CK(conv<7>(s, x, ch, Tl, h->w(ti), h->w(ti + 1), d_wav, 1, 1, 0));
  return MVB_OK;
}

// ---- batched decode ------------------------------------------------------------------------------------------------------
// Batch workspace (caller-owned, separate from the handle's): segment table | three activation buffers | LSTM
// pre-activations | h exchange [2][max_batch][H] | barrier word, all sized for max_total_frames concatenated frames.
struct VocBatchLayout { size_t seg, A, B, C, pre, h, bar, total; };

static VocBatchLayout voc_batch_layout(const mvb_voc_config* c, int max_batch, int max_total_frames) {
  const size_t maxelems = voc_max_elems(c, (size_t)max_total_frames);
  const size_t top = (size_t)(c->n_filters << c->n_ratios);
  VocBatchLayout L;
  WsBump ws;
  L.seg = ws.take((size_t)VOC_MAX_BATCH * sizeof(Seg));
  L.A = ws.take(maxelems * 4); L.B = ws.take(maxelems * 4); L.C = ws.take(maxelems * 4);
  L.pre = ws.take(4 * top * (size_t)max_total_frames * 4);
  L.h = ws.take(2 * (size_t)max_batch * top * 4);
  L.bar = ws.take(256);
  L.total = ws.end;
  return L;
}

static int voc_batch_capacity(int max_batch, int max_total_frames) {
  if (max_batch < 1 || max_batch > VOC_MAX_BATCH)
    return mvb::set_error(MVB_ERR_ARG, "vocoder batch: max_batch %d out of range [1, %d]", max_batch, VOC_MAX_BATCH);
  if (max_total_frames < 8) return mvb::set_error(MVB_ERR_ARG, "vocoder batch: max_total_frames %d < 8", max_total_frames);
  return MVB_OK;
}

extern "C" size_t mvb_voc_batch_workspace_bytes(const mvb_voc_config* c, int32_t max_batch, int32_t max_total_frames) {
  if (voc_validate(c) || voc_batch_capacity(max_batch, max_total_frames)) return 0;
  return voc_batch_layout(c, max_batch, max_total_frames).total;
}

// Validates a batch (nothing is launched on failure) and uploads its segment table; *T_max = the longest utterance.
static int voc_batch_begin(const mvb_voc* h, int n, const int32_t* d_codes, const int32_t* T, void* d_ws, int max_batch,
                           int max_total_frames, const void* d_out, cudaStream_t s, const VocBatchLayout& L, int* T_max) {
  if (!h || !d_codes || !T || !d_ws || !d_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (int e = voc_batch_capacity(max_batch, max_total_frames)) return e;
  if (n < 1 || n > max_batch) return mvb::set_error(MVB_ERR_ARG, "vocoder batch: %d utterances, capacity %d", n, max_batch);
  Seg segs[VOC_MAX_BATCH];
  long long total = 0;
  int tmax = 0;
  for (int i = 0; i < n; ++i) {
    if (T[i] < 8 || T[i] > h->cfg.max_frames)
      return mvb::set_error(MVB_ERR_ARG, "vocoder batch: utterance %d: frame count %d out of range [8, %d]", i, T[i], h->cfg.max_frames);
    segs[i] = Seg{T[i], (int)total};
    total += T[i];
    if (T[i] > tmax) tmax = T[i];
  }
  if (total > max_total_frames)
    return mvb::set_error(MVB_ERR_ARG, "vocoder batch: %lld frames in all, capacity %d", total, max_total_frames);
  MVB_CK(cudaMemcpyAsync(reinterpret_cast<char*>(d_ws) + L.seg, segs, n * sizeof(Seg), cudaMemcpyHostToDevice, s));
  *T_max = tmax;
  return MVB_OK;
}

template <int K>
static cudaError_t conv_b(cudaStream_t s, const float* x, int Cin, const Seg* segs, int n, int T_max, int m, const float* w,
                          const float* b, float* y, int Cout, int elu, int acc) {
  k_conv1d_b<K><<<dim3((T_max * m + 255) / 256, (Cout + 31) / 32, n), 256, 0, s>>>(x, Cin, segs, m, w, b, y, Cout, elu, acc);
  return cudaGetLastError();
}

extern "C" int mvb_voc_decode_latent_batch(mvb_voc* h, int32_t n, const int32_t* d_codes, const int32_t* T, void* d_batch_ws,
                                           int32_t max_batch, int32_t max_total_frames, float* d_latent, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  const VocBatchLayout L = h ? voc_batch_layout(&h->cfg, max_batch, max_total_frames) : VocBatchLayout{};
  int T_max = 0;
  if (int e = voc_batch_begin(h, n, d_codes, T, d_batch_ws, max_batch, max_total_frames, d_latent, s, L, &T_max)) return e;
  const Seg* segs = reinterpret_cast<const Seg*>(reinterpret_cast<char*>(d_batch_ws) + L.seg);
  k_rvq_decode_b<<<dim3((T_max + 31) / 32, 1, n), 128, 0, s>>>(d_codes, h->cfg.n_q, segs, h->books_dev, h->cfg.hidden, d_latent);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

// The launch sequence of mvb_voc_decode, each launch over all n utterances.
extern "C" int mvb_voc_decode_batch(mvb_voc* h, int32_t n, const int32_t* d_codes, const int32_t* T, void* d_batch_ws,
                                    int32_t max_batch, int32_t max_total_frames, float* d_wav, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  const VocBatchLayout L = h ? voc_batch_layout(&h->cfg, max_batch, max_total_frames) : VocBatchLayout{};
  int T_max = 0;
  if (int e = voc_batch_begin(h, n, d_codes, T, d_batch_ws, max_batch, max_total_frames, d_wav, s, L, &T_max)) return e;
  const mvb_voc_config& c = h->cfg;
  const int top = c.n_filters << c.n_ratios;
  if (int e = lstm_b_check_coresident(top, n)) return e;
  char* ws = reinterpret_cast<char*>(d_batch_ws);
  const Seg* segs = reinterpret_cast<const Seg*>(ws + L.seg);
  float *A = (float*)(ws + L.A), *B = (float*)(ws + L.B), *Cc = (float*)(ws + L.C), *pre = (float*)(ws + L.pre);
  float* hbuf = (float*)(ws + L.h);
  unsigned* bar = (unsigned*)(ws + L.bar);
  int ti = c.n_q;
  k_rvq_decode_b<<<dim3((T_max + 31) / 32, 1, n), 128, 0, s>>>(d_codes, c.n_q, segs, h->books_dev, c.hidden, A);
  MVB_CK(cudaGetLastError());
  MVB_CK(conv_b<7>(s, A, c.hidden, segs, n, T_max, 1, h->w(ti), h->w(ti + 1), B, top, 0, 0));      // conv_in
  ti += 2;
  const float* lin = B;
  float* louts[2] = {A, Cc};
  for (int l = 0; l < 2; ++l) {
    MVB_CK(conv_b<1>(s, lin, top, segs, n, T_max, 1, h->w(ti), h->w(ti + 2), pre, 4 * top, 0, 0));
    MVB_CK(cudaMemsetAsync(bar, 0, 4, s));
    k_lstm_layer_b<<<top / 4, 128, lstm_b_smem(top, n), s>>>(pre, h->w(ti + 1), top, segs, n, T_max, hbuf, bar, louts[l],
                                                             l == 1 ? B : nullptr);
    MVB_CK(cudaGetLastError());
    lin = louts[l];
    ti += 3;
  }
  float* x = Cc;
  float* f1 = A;
  float* f2 = B;
  int ch = top, m = 1;
  for (int i = 0; i < c.n_ratios; ++i) {
    const int r = c.ratios[i], co = ch / 2;
    const size_t smem = (size_t)(16 * 33 + 16 * 32 * 2 * r) * 4;
    k_convtr1d_b<<<dim3((T_max * m + 31) / 32, (co + 31) / 32, n), 256, smem, s>>>(x, ch, segs, m, h->w(ti), h->w(ti + 1), f1, co, r);
    MVB_CK(cudaGetLastError());
    m *= r; ch = co;
    MVB_CK(conv_b<3>(s, f1, ch, segs, n, T_max, m, h->w(ti + 2), h->w(ti + 3), f2, ch / c.compress, 1, 0));
    MVB_CK(conv_b<1>(s, f1, ch, segs, n, T_max, m, h->w(ti + 6), h->w(ti + 7), x, ch, 0, 0));
    MVB_CK(conv_b<1>(s, f2, ch / c.compress, segs, n, T_max, m, h->w(ti + 4), h->w(ti + 5), x, ch, 1, 1));
    ti += 8;
  }
  MVB_CK(conv_b<7>(s, x, ch, segs, n, T_max, m, h->w(ti), h->w(ti + 1), d_wav, 1, 1, 0));
  return MVB_OK;
}

extern "C" int mvb_voc_op_test(int32_t op, const float* d_x, int32_t Cin, int32_t T, const float* d_w, const float* d_b,
                               int32_t Cout, int32_t k, int32_t elu_in, int32_t accumulate, const float* d_skip, float* d_y,
                               void* stream) {
  if (!d_x || !d_w || !d_y) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (Cin < 1 || T < 1) return mvb::set_error(MVB_ERR_ARG, "mvb_voc_op_test: bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  if (op == 0) {
    if (Cout < 1) return mvb::set_error(MVB_ERR_ARG, "mvb_voc_op_test: bad shape");
    if (k == 1) MVB_CK(conv<1>(s, d_x, Cin, T, d_w, d_b, d_y, Cout, elu_in, accumulate));
    else if (k == 3) MVB_CK(conv<3>(s, d_x, Cin, T, d_w, d_b, d_y, Cout, elu_in, accumulate));
    else if (k == 7) MVB_CK(conv<7>(s, d_x, Cin, T, d_w, d_b, d_y, Cout, elu_in, accumulate));
    else return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_voc_op_test: conv kernel size %d", k);
  } else if (op == 1) {
    if (Cout < 1 || !d_b) return mvb::set_error(MVB_ERR_ARG, "mvb_voc_op_test: bad shape or null bias");
    if (k < 1 || k > 8) return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_voc_op_test: upsampling ratio %d", k);
    MVB_CK(convtr(s, d_x, Cin, T, d_w, d_b, d_y, Cout, k));
  } else if (op == 2) {
    const int H = Cin;
    if (H % 32 || lstm_smem(H) > (size_t)LSTM_SMEM_LIMIT) return mvb::set_error(MVB_ERR_UNSUPPORTED, "LSTM width %d unsupported", H);
    if (int e = lstm_check_coresident(H)) return e;
    WsBump ws;
    const size_t o_h = ws.take((size_t)2 * H * 4), o_bar = ws.take(4);
    char* buf = nullptr;
    MVB_CK(cudaMalloc(&buf, ws.end));
    cudaError_t e = lstm(s, d_x, d_w, H, T, reinterpret_cast<float*>(buf + o_h), reinterpret_cast<unsigned*>(buf + o_bar), d_y, d_skip);
    const cudaError_t es = cudaStreamSynchronize(s);   // (also on an error path: the buffer is freed only once unused)
    cudaFree(buf);
    if (e == cudaSuccess) e = es;
    if (e != cudaSuccess) return mvb::set_error(MVB_ERR_CUDA, "mvb_voc_op_test: %s", cudaGetErrorString(e));
    return MVB_OK;
  } else {
    return mvb::set_error(MVB_ERR_ARG, "mvb_voc_op_test: op %d", op);
  }
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}
