// Kernels and launch helpers shared by the two directions of the EnCodec-24 kHz codec: the decoder (vocoder.cu) and the
// encoder (encoder.cu).  Operator semantics follow transformers' modeling_encodec.py (cited per kernel); fp32 throughout.
//
// Activations are [C][T] fp32 per utterance (time contiguous).  Every kernel runs n <= 32 utterances in one launch,
// passed by value as a segment list {T_i, off_i, len_i}: a layer with C channels at m samples per frame holds utterance
// i as a [C, T_i m] block starting at element C off_i m (off_i = T_0 + ... + T_{i-1}).  blockIdx.z is the utterance and
// tiles past its end return, so every utterance is computed exactly as it is alone.
//
// len_i is the utterance's valid length at the launch's rate, capped at the block length T_i m: the encoder's levels
// hold ceil(L_i m / 320) valid samples of an L_i-sample input in a block of T_i m = ceil(L_i / 320) m.  The decoder's
// blocks are full (SEG_WHOLE).  A kernel reads nothing past the valid length (it pads as the reference pads a tensor of
// that length) and writes only valid outputs.
#pragma once
#include <cuda_runtime.h>

#include <climits>

#include "common.cuh"
#include "host.cuh"

namespace {

using mvb::red_release_inc;
using mvb::wait_counter;

constexpr int CODEC_MAX_BATCH = 32;
constexpr int SEG_WHOLE = INT_MAX;      // len of a segment whose every block sample is valid
struct Seg { int T, off, len; };
struct Segs { Seg s[CODEC_MAX_BATCH]; };   // a kernel parameter (384 B): indexing it needs no device table

__device__ __forceinline__ float elu1(float v) { return v > 0.f ? v : expm1f(v); }

// Reflect padding of a sequence of V valid samples as EncodecConv1d._pad1d applies it for a padding of at most max_pad
// samples on either side: t < 0 reflects to -t, t >= V to 2 (V - 1) - t.  When V <= max_pad, _pad1d first extends the
// sequence with zeros to max_pad + 1 samples, reflects that and trims the extension again: the reflection is then about
// max_pad instead of V - 1, and every index that lands at or past V reads zero.  Returns the source index, or -1 for a
// zero (also for t past the padding, which no valid output reads).
__device__ __forceinline__ int reflect_src(int t, int V, int max_pad) {
  const int Vr = V > max_pad ? V : max_pad + 1;
  if (t < 0) t = -t;
  else if (t >= Vr) t = 2 * (Vr - 1) - t;
  return (t >= 0 && t < V) ? t : -1;
}

// Causal Conv1d, stride 1, dilation 1, reflect padding of K-1 samples on the left (EncodecConv1d, causal branch),
// optional ELU on the input (the nn.ELU() that precedes the conv in the stack) and optional accumulation into y
// (residual / shortcut sum of EncodecResnetBlock).  Tile: 32 output channels x 256 samples, 16 input channels per pass.
// Input and output at m samples per frame: x [Cin, T] -> y [Cout, T] per utterance, T = T_i m, of which the first
// V = min(len_i, T) are valid.  Output t < V reads inputs t-K+1 .. t and the reflection of inputs 1 .. K-1 (reflect_src:
// zeros past V when V <= K - 1); outputs t >= V are not written.
template <int K>
__global__ void __launch_bounds__(256) k_conv1d(const float* __restrict__ x, int Cin, Segs segs, int m, const float* __restrict__ w,
                                                const float* __restrict__ bias, float* __restrict__ y, int Cout, int elu_in,
                                                int accumulate) {
  constexpr int CI = 16, TT = 256, CO = 32;
  __shared__ float xs[CI][TT + K - 1 + 1];
  __shared__ float ws[CO][CI][K];
  const Seg g = segs.s[blockIdx.z];
  const int T = g.T * m, V = min(g.len, T), t0 = blockIdx.x * TT, co0 = blockIdx.y * CO;
  if (t0 >= V) return;
  const float* __restrict__ xb = x + (size_t)g.off * m * Cin;
  float* __restrict__ yb = y + (size_t)g.off * m * Cout;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;    // 64 time groups of 4 samples x 4 groups of 8 channels
  // 128-bit loads and stores need T % 4 == 0 and 16-byte aligned sequence bases (a segment may start anywhere)
  const bool vec = (T & 3) == 0 && ((reinterpret_cast<uintptr_t>(xb) | reinterpret_cast<uintptr_t>(yb)) & 15) == 0;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int c0 = 0; c0 < Cin; c0 += CI) {
    __syncthreads();
    // line buffer: samples t0-(K-1) .. t0+TT-1 of 16 channels.  The TT-sample body is streamed with 128-bit loads
    // (rows are 16-byte aligned when T % 4 == 0, which holds for every layer at 4 or more samples per frame); a float4
    // that straddles V carries samples past it, which only outputs past V read.  The K-1 halo samples in front are
    // loaded one by one through reflect_src.
    if (vec) {
      for (int i = threadIdx.x; i < CI * (TT / 4); i += 256) {
        const int ci = i / (TT / 4), q4 = i - ci * (TT / 4);
        const int t = t0 + 4 * q4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c0 + ci < Cin && t < V) {          // T % 4 == 0: a float4 that starts before V ends inside the block
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
      const int t = t0 + tt - (K - 1);
      const int src = t < 0 ? reflect_src(t, V, K - 1) : (t < V ? t : -1);
      float v = 0.f;
      if (c0 + ci < Cin && src >= 0) {
        v = xb[(size_t)(c0 + ci) * T + src];
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
    if (vec && tb + 3 < V) {                   // 128-bit coalesced store of the thread's 4 consecutive samples
      float4* o = reinterpret_cast<float4*>(yb + (size_t)co * T + tb);
      float4 v = make_float4(acc[i][0] + bv, acc[i][1] + bv, acc[i][2] + bv, acc[i][3] + bv);
      if (accumulate) { const float4 p = *o; v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w; }
      *o = v;
      continue;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int t = t0 + tx * 4 + j;
      if (t < V) {
        float* o = yb + (size_t)co * T + t;
        const float v = acc[i][j] + bv;
        *o = accumulate ? *o + v : v;
      }
    }
  }
}

// One LSTM layer (EncodecLSTM: nn.LSTM, gate order i, f, g, o, zero initial state) for n <= 32 sequences, persistent over
// time: one grid barrier per step of the longest sequence.  CTA c owns hidden units [4c, 4c+4) and holds their 16 W_hh
// rows in shared memory, loaded once; each step it computes those 16 gate rows for every sequence still running
// (t < T_i) and the finished ones stop writing.  h_{t-1} is exchanged through global memory.  Each pre-activation is
// summed by 8 lanes x H/8 consecutive products, then xor-shuffles 4 / 2 / 1, in the same order for every n.  Shared
// memory rows are padded by one float per H/8 segment: the 8 lanes of a row and the 4 rows of a warp then read 32
// different banks.  pre[row][t] = W_ih x_t + b_ih + b_hh is computed beforehand by k_conv1d<1>; the skip connection of
// EncodecLSTM (output + input) is fused into the last layer's store.  The LSTM runs at one sample per frame, where every
// block sample is valid.
// pre: per sequence [4H, T_i] at 4H off_i; out / skip: [H, T_i] at H off_i; hbuf [2][n][H].
__host__ __device__ constexpr int lstm_ld(int H) { return H + 8; }

__global__ void __launch_bounds__(128) k_lstm_layer(const float* __restrict__ pre, const float* __restrict__ whh, int H, Segs segs,
                                                    int n, int T_max, float* __restrict__ hbuf, unsigned* bar, float* __restrict__ out,
                                                    const float* __restrict__ skip) {
  extern __shared__ float sm[];
  const int seg = H / 8, ld = lstm_ld(H);
  float* wsm = sm;                 // [16][ld]
  float* hs = sm + 16 * ld;        // [round_up(n, 4)][ld]
  __shared__ float gates[CODEC_MAX_BATCH][16];
  __shared__ int Ts[CODEC_MAX_BATCH], offs[CODEC_MAX_BATCH];
  const int cta = blockIdx.x, tid = threadIdx.x;
  const int u0 = cta * 4;
  const int n4 = (n + 3) & ~3;
  auto at = [seg](int k) { const int p = k / seg; return p * (seg + 1) + (k - p * seg); };   // padded column of k
  for (int i = tid; i < 16 * H; i += 128) {
    const int r = i / H, k = i - r * H;
    const int grow = (r >> 2) * H + u0 + (r & 3);
    wsm[r * ld + at(k)] = whh[(size_t)grow * H + k];
  }
  if (tid < n) { Ts[tid] = segs.s[tid].T; offs[tid] = segs.s[tid].off; }
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

Segs one_segment(int T, int len = SEG_WHOLE) {
  Segs g{};
  g.s[0] = Seg{T, 0, len};
  return g;
}

// k_lstm_layer: W_hh slice + h of round_up(n, 4) sequences, rows padded to lstm_ld(H), under the 100 KB opt-in set below
constexpr int LSTM_SMEM_LIMIT = 100 * 1024;
size_t lstm_smem(int H, int n) { return (size_t)(16 + ((n + 3) & ~3)) * lstm_ld(H) * 4; }

int lstm_set_smem_limit() {
  static mvb::PerDeviceOnce attr;
  if (attr.pending()) {
    MVB_CK(cudaFuncSetAttribute(k_lstm_layer, cudaFuncAttributeMaxDynamicSharedMemorySize, LSTM_SMEM_LIMIT));
    attr.mark();
  }
  return MVB_OK;
}

// The H / 4 CTAs of one LSTM layer meet at a grid-wide barrier every step, so all of them must be resident at once on
// the current device; a layer that cannot be is rejected instead of launched (it would wait forever).
int lstm_check_coresident(int H, int n) {
  if (int e = lstm_set_smem_limit()) return e;
  int dev = 0, n_sm = 0, per_sm = 0;
  if (int e = mvb::current_device(&dev, &n_sm)) return e;
  MVB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_lstm_layer, 128, lstm_smem(H, n)));
  if (H / 4 > per_sm * n_sm)
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "LSTM width %d: %d CTAs cannot be co-resident (%d per SM x %d SMs)", H, H / 4,
                          per_sm, n_sm);
  return MVB_OK;
}

// Launches over n segments, T_max = the longest; activations at m samples per frame.
template <int K>
cudaError_t conv(cudaStream_t s, const float* x, int Cin, const Segs& segs, int n, int T_max, int m, const float* w,
                 const float* b, float* y, int Cout, int elu, int acc) {
  k_conv1d<K><<<dim3((T_max * m + 255) / 256, (Cout + 31) / 32, n), 256, 0, s>>>(x, Cin, segs, m, w, b, y, Cout, elu, acc);
  return cudaGetLastError();
}

// One LSTM layer; the caller has checked lstm_check_coresident(H, n) and set the shared-memory limit.
cudaError_t lstm(cudaStream_t s, const float* pre, const float* whh, int H, const Segs& segs, int n, int T_max, float* hbuf,
                 unsigned* bar, float* out, const float* skip) {
  cudaError_t e = cudaMemsetAsync(bar, 0, 4, s);
  if (e != cudaSuccess) return e;
  k_lstm_layer<<<H / 4, 128, lstm_smem(H, n), s>>>(pre, whh, H, segs, n, T_max, hbuf, bar, out, skip);
  return cudaGetLastError();
}

}  // namespace
