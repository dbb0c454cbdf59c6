// EnCodec-24 kHz encode path: waveform -> SEANet encoder -> residual vector quantiser -> codes, the other direction of
// vocoder.cu.  This is what `EncodecDecoder.get_tokens` (fam/llm/decoders.py:49-64) and the fine-tuning loader's
// `_extract_encodec_tokens` (fam/llm/loaders/training_data.py:98-112) compute through `codec_model.encode`, i.e.
// transformers' EncodecModel.encode with the default EncodecConfig (normalize=False, one chunk, causal, reflect padding).
// fp32 throughout.
//
// Stack (EncodecEncoder, modeling_encodec.py:285-313): conv_in 1 -> 32 (k 7); per ratio of (2, 4, 5, 8) at C = 32 .. 256:
// residual block (ELU, k3 C -> C/2, ELU, k1 C/2 -> C, plus a 1x1 shortcut), ELU + strided conv C -> 2C (k 2r, stride r);
// 2-layer LSTM(512) with skip; ELU + conv 512 -> 128 (k 7).  Then RVQ encode over n_q codebooks.
//
// An utterance of L samples has F = ceil(L / 320) frames.  It is laid out as the decoder lays it out (codec.cuh: a level
// at m samples per frame holds it as [C, F m] at C off m), and a level's valid length is len = ceil(L m / 320): each
// EncodecConv1d pads a tensor of that length and emits ceil(len / stride) samples.  Every kernel takes len from the
// segment list, so the samples between len and the block end are never read into a valid output.
#include <cuda_runtime.h>

#include <vector>

#include "codec.cuh"
#include "common.cuh"
#include "host.cuh"

using namespace mvb;

namespace {

constexpr int ENC_BINS = 1024;   // codebook rows

// Packed waveforms -> block layout: utterance i's len_i samples, stored at L_0 + ... + L_{i-1}, go to [T_i hop] at
// off_i hop.  Only the len_i samples are written.
__global__ void __launch_bounds__(256) k_pack_wav(const float* __restrict__ x, Segs segs, int hop, float* __restrict__ y) {
  const Seg g = segs.s[blockIdx.z];
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= g.len) return;
  size_t in = 0;
  for (int i = 0; i < (int)blockIdx.z; ++i) in += segs.s[i].len;
  y[(size_t)g.off * hop + t] = x[in + t];
}

// Causal strided Conv1d (EncodecConv1d with kernel 2S, stride S: the encoder's downsampling layers) with the preceding
// ELU fused, bias.  Input at m samples per frame, output at m / S: x [Cin, T] with V = min(len, T) valid ->
// y [Cout, T / S], of which the Vo = ceil(V / S) valid outputs are written.  Output o reads p[o S .. o S + 2S - 1] of the
// padded input p[j] = x[j - S]: S samples of reflect padding on the left and Vo S - V on the right, both resolved by
// reflect_src(t, V, S) (S is the larger of the two paddings).
// Tile: 32 output channels x 256 outputs, CI input channels per pass.  The line buffer holds the tile's window of
// 256 S + S input samples in polyphase order xs[ci][r][q] (window sample l = q S + r), so tap k of output o lies at
// (k % S, o + k / S) and the 32 lanes of a warp, which own consecutive outputs, read consecutive words.  Thread: 8
// channels x the outputs tx + 64 j, j = 0..3.  The window body is streamed with 128-bit loads wherever 4 samples lie
// inside V; the halo and the right padding go through reflect_src one sample at a time.
// Summation order of every output (the tests derive their bound from it): one fmaf chain from 0 over the input channels
// in ascending order, within a channel the taps k = 0, S, 1, S + 1, ..., S - 1, 2S - 1; then one add of the bias.
template <int S>
__global__ void __launch_bounds__(256) k_conv1d_down(const float* __restrict__ x, int Cin, Segs segs, int m,
                                                     const float* __restrict__ w, const float* __restrict__ bias,
                                                     float* __restrict__ y, int Cout) {
  constexpr int TO = 256, CO = 32, K = 2 * S, Q = TO + 1, WIN = TO * S + S;
  constexpr int CI = S == 2 ? 16 : S == 4 ? 8 : 4;          // line buffer CI x WIN floats <= 33 KB
  __shared__ float xs[CI][S][Q];
  __shared__ float ws[CO][CI][K];
  const Seg g = segs.s[blockIdx.z];
  const int T = g.T * m, V = min(g.len, T), Vo = (V + S - 1) / S, To = T / S;
  const int o0 = blockIdx.x * TO, co0 = blockIdx.y * CO;
  if (o0 >= Vo) return;
  const float* __restrict__ xb = x + (size_t)g.off * m * Cin;
  float* __restrict__ yb = y + (size_t)g.off * m / S * Cout;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int t_start = o0 * S - S;                            // input time of window sample 0
  const bool vec = (T & 3) == 0 && (reinterpret_cast<uintptr_t>(xb) & 15) == 0;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int c0 = 0; c0 < Cin; c0 += CI) {
    __syncthreads();
    if (vec) {
      // body: window samples S .. WIN - 1 (times o0 S ..), 16-byte aligned because o0 S % 4 == 0 and T % 4 == 0
      for (int i = threadIdx.x; i < CI * (TO * S / 4); i += 256) {
        const int ci = i / (TO * S / 4), q4 = i - ci * (TO * S / 4);
        const int t = o0 * S + 4 * q4, l = S + 4 * q4;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (c0 + ci < Cin) {
          const float* row = xb + (size_t)(c0 + ci) * T;
          if (t + 3 < V) {
            const float4 f = *reinterpret_cast<const float4*>(row + t);
            v[0] = elu1(f.x); v[1] = elu1(f.y); v[2] = elu1(f.z); v[3] = elu1(f.w);
          } else {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int src = reflect_src(t + e, V, S);
              v[e] = src >= 0 ? elu1(row[src]) : 0.f;
            }
          }
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) xs[ci][(l + e) % S][(l + e) / S] = v[e];
      }
    }
    for (int i = threadIdx.x; i < CI * (vec ? S : WIN); i += 256) {
      const int span = vec ? S : WIN;
      const int ci = i / span, l = i - ci * span;
      const int src = reflect_src(t_start + l, V, S);
      xs[ci][l % S][l / S] = (c0 + ci < Cin && src >= 0) ? elu1(xb[(size_t)(c0 + ci) * T + src]) : 0.f;
    }
    for (int i = threadIdx.x; i < CO * CI * K; i += 256) {
      const int co = i / (CI * K), r = i - co * (CI * K), ci = r / K, k = r - ci * K;
      ws[co][ci][k] = (co0 + co < Cout && c0 + ci < Cin) ? w[((size_t)(co0 + co) * Cin + c0 + ci) * K + k] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int ci = 0; ci < CI; ++ci) {
#pragma unroll
      for (int r = 0; r < S; ++r) {
        float xa[4], xc[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { xa[j] = xs[ci][r][tx + 64 * j]; xc[j] = xs[ci][r][tx + 64 * j + 1]; }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float w0 = ws[ty * 8 + i][ci][r], w1 = ws[ty * 8 + i][ci][r + S];
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(w1, xc[j], fmaf(w0, xa[j], acc[i][j]));
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int co = co0 + ty * 8 + i;
    if (co >= Cout) continue;
    const float bv = bias[co];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = o0 + tx + 64 * j;
      if (o < Vo) yb[(size_t)co * To + o] = acc[i][j] + bv;
    }
  }
}

// |e_j|^2 of every codebook row, summed in double and rounded once to fp32 (create time): nrm [n_q][ENC_BINS].
__global__ void k_sq_norms(const float* const* __restrict__ books, int dim, float* __restrict__ nrm) {
  const int q = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ENC_BINS) return;
  const float* e = books[q] + (size_t)j * dim;
  double s = 0.0;
  for (int d = 0; d < dim; ++d) s += (double)e[d] * (double)e[d];
  nrm[(size_t)q * ENC_BINS + j] = (float)s;
}

// Residual vector quantiser, encode (EncodecResidualVectorQuantizer.encode :424-438 over
// EncodecEuclideanCodebook.quantize :364-369): for q = 0 .. n_q - 1, idx = argmin_j (|e_j|^2 - 2 r . e_j) over the
// ENC_BINS rows of codebook q -- the reference's |r|^2 term is the same for every j -- with the lowest j on exact ties
// (torch.max returns the first maximum); then r -= e_idx in fp32.  r starts as the frame's embedding and stays in shared
// memory across the n_q codebooks.
// One CTA = 32 frames of one segment.  Lane = frame; warp w scores rows 4w .. 4w + 3 of each 32-row chunk of the
// codebook staged in shared memory, chunks in ascending order, and keeps its first best; the 8 warps' bests are then
// merged by (score, index).  Score of row j: dot = one fmaf chain from 0 over d = 0 .. dim - 1 in ascending order,
// s = nrm[j] - 2 dot (the doubling is exact: one rounding).
// emb [dim, T_i] at dim off_i -> codes int32 [n_q, T_i] at n_q off_i; res_out (optional) [dim, T_i] at dim off_i: the
// residual after the last codebook.  dim <= 128.
__global__ void __launch_bounds__(256) k_rvq_encode(const float* __restrict__ emb, int dim, Segs segs,
                                                    const float* const* __restrict__ books, const float* __restrict__ nrm, int n_q,
                                                    int* __restrict__ codes, float* __restrict__ res_out) {
  constexpr int FT = 32, RC = 32, DP = 132;
  __shared__ __align__(16) float r[FT][DP];
  __shared__ __align__(16) float e[RC][128];
  __shared__ float best_s[8][FT];
  __shared__ int best_j[8][FT], pick[FT];
  // the segment goes through shared memory: read from the parameter directly, ptxas spills it (as in k_convtr1d)
  __shared__ Seg gs;
  if (threadIdx.x == 0) gs = segs.s[blockIdx.z];
  __syncthreads();
  const Seg g = gs;
  const int T = g.T, t0 = blockIdx.x * FT;
  if (t0 >= T) return;
  emb += (size_t)dim * g.off;
  codes += (size_t)n_q * g.off;
  const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
  const int d4 = (dim + 3) >> 2;           // rows zero-padded to a multiple of 4 (zeros add exact zeros to the chain)
  for (int i = tid; i < FT * d4 * 4; i += 256) {
    const int d = i / FT, f = i - d * FT;
    r[f][d] = (d < dim && t0 + f < T) ? emb[(size_t)d * T + t0 + f] : 0.f;
  }
  for (int q = 0; q < n_q; ++q) {
    const float* __restrict__ book = books[q];
    const float* __restrict__ nq = nrm + (size_t)q * ENC_BINS;
    float bs = INFINITY;
    int bj = 0;
    for (int c = 0; c < ENC_BINS; c += RC) {
      __syncthreads();
      for (int i = tid; i < RC * d4 * 4; i += 256) {
        const int row = i / (d4 * 4), d = i - row * (d4 * 4);
        e[row][d] = d < dim ? book[(size_t)(c + row) * dim + d] : 0.f;
      }
      __syncthreads();
      // four rows per thread, each its own fmaf chain over d ascending
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      const float4* rp = reinterpret_cast<const float4*>(&r[lane][0]);
      const float4* e0 = reinterpret_cast<const float4*>(&e[wp * 4][0]);
#pragma unroll 4
      for (int k4 = 0; k4 < d4; ++k4) {
        const float4 rv = rp[k4];
        const float4 v0 = e0[k4], v1 = e0[32 + k4], v2 = e0[64 + k4], v3 = e0[96 + k4];
        a0 = fmaf(rv.w, v0.w, fmaf(rv.z, v0.z, fmaf(rv.y, v0.y, fmaf(rv.x, v0.x, a0))));
        a1 = fmaf(rv.w, v1.w, fmaf(rv.z, v1.z, fmaf(rv.y, v1.y, fmaf(rv.x, v1.x, a1))));
        a2 = fmaf(rv.w, v2.w, fmaf(rv.z, v2.z, fmaf(rv.y, v2.y, fmaf(rv.x, v2.x, a2))));
        a3 = fmaf(rv.w, v3.w, fmaf(rv.z, v3.z, fmaf(rv.y, v3.y, fmaf(rv.x, v3.x, a3))));
      }
      const int j0 = c + wp * 4;
      const float s0 = nq[j0] - 2.f * a0, s1 = nq[j0 + 1] - 2.f * a1, s2 = nq[j0 + 2] - 2.f * a2, s3 = nq[j0 + 3] - 2.f * a3;
      if (s0 < bs) { bs = s0; bj = j0; }
      if (s1 < bs) { bs = s1; bj = j0 + 1; }
      if (s2 < bs) { bs = s2; bj = j0 + 2; }
      if (s3 < bs) { bs = s3; bj = j0 + 3; }
    }
    best_s[wp][lane] = bs;
    best_j[wp][lane] = bj;
    __syncthreads();
    if (tid < FT) {
      float s = best_s[0][tid];
      int j = best_j[0][tid];
      for (int w = 1; w < 8; ++w) {
        const float sw = best_s[w][tid];
        const int jw = best_j[w][tid];
        if (sw < s || (sw == s && jw < j)) { s = sw; j = jw; }
      }
      pick[tid] = j;
      if (t0 + tid < T) codes[(size_t)q * T + t0 + tid] = j;
    }
    __syncthreads();
    for (int i = tid; i < FT * dim; i += 256) {
      const int f = i / dim, d = i - f * dim;
      r[f][d] = r[f][d] - book[(size_t)pick[f] * dim + d];
    }
  }
  if (res_out) {
    __syncthreads();
    res_out += (size_t)dim * g.off;
    for (int i = tid; i < FT * dim; i += 256) {
      const int d = i / FT, f = i - d * FT;
      if (t0 + f < T) res_out[(size_t)d * T + t0 + f] = r[f][d];
    }
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// Encoder workspace for max_batch utterances of max_total_frames frames in all: three activation buffers | LSTM
// pre-activations | embeddings | h exchange [2][max_batch][H] | barrier word.  A batch workspace is this layout; the
// handle's own workspace is this layout at (1, max_frames) followed by the codebook pointer table and |e|^2 [n_q][1024].
struct EncLayout { size_t A, B, C, pre, emb, h, bar, total; };
struct EncBufs { float *A, *B, *C, *pre, *emb, *hbuf; unsigned* bar; };

struct mvb_enc {
  mvb_enc_config cfg;
  int hop;                      // samples per frame: prod(ratios)
  const char* arena;
  std::vector<uint64_t> off;
  EncBufs bufs;                 // in the handle's workspace: mvb_enc_encode
  const float** books_dev;
  float* norms;
  const float* w(int i) const { return reinterpret_cast<const float*>(arena + off[i]); }
};

// tensor order in the arena (fp32, weight norm folded by the loader):
//   codebooks[n_q] | conv_in {w,b} | per level, ratios in reverse: res.c1 {w,b}, res.c2 {w,b}, res.shortcut {w,b},
//   down {w,b} | lstm l0 {w_ih, w_hh, b_ih+b_hh} | lstm l1 {...} | conv_out {w,b}
static int enc_n_tensors(const mvb_enc_config* c) { return c->n_q + 2 + c->n_ratios * 8 + 6 + 2; }

static int enc_hop(const mvb_enc_config* c) {
  int hop = 1;
  for (int i = 0; i < c->n_ratios; ++i) hop *= c->ratios[i];
  return hop;
}

static EncLayout enc_layout(const mvb_enc_config* c, int max_batch, int max_total_frames) {
  const size_t T = (size_t)max_total_frames;
  // elements per frame of the largest activation over the downsampling levels (the packed input is 1 x hop)
  size_t m = (size_t)enc_hop(c), ch = (size_t)c->n_filters, per_frame = ch * m;
  for (int i = c->n_ratios - 1; i >= 0; --i) {
    m /= c->ratios[i];
    ch *= 2;
    if (ch * m > per_frame) per_frame = ch * m;
  }
  const size_t top = (size_t)(c->n_filters << c->n_ratios);
  EncLayout L;
  WsBump ws;
  L.A = ws.take(per_frame * T * 4); L.B = ws.take(per_frame * T * 4); L.C = ws.take(per_frame * T * 4);
  L.pre = ws.take(4 * top * T * 4);
  L.emb = ws.take((size_t)c->hidden * T * 4);
  L.h = ws.take(2 * (size_t)max_batch * top * 4);
  L.bar = ws.take(256);
  L.total = ws.end;
  return L;
}

static EncBufs enc_bufs(void* d_ws, const EncLayout& L) {
  char* ws = reinterpret_cast<char*>(d_ws);
  return EncBufs{(float*)(ws + L.A), (float*)(ws + L.B), (float*)(ws + L.C), (float*)(ws + L.pre), (float*)(ws + L.emb),
                 (float*)(ws + L.h), (unsigned*)(ws + L.bar)};
}

constexpr size_t ENC_BOOKS_BYTES = 64 * sizeof(void*);   // codebook pointer table, after enc_layout(1, max_frames)
static size_t enc_norms_bytes(const mvb_enc_config* c) { return (size_t)c->n_q * ENC_BINS * 4; }

static int enc_validate(const mvb_enc_config* c) {
  if (!c) return mvb::set_error(MVB_ERR_ARG, "null config");
  if (c->n_ratios < 1 || c->n_ratios > 8 || c->n_q < 1 || c->n_q > 32 || c->hidden < 1 || c->n_filters < 1 || c->compress < 1)
    return mvb::set_error(MVB_ERR_ARG, "bad codec shape");
  if (c->hidden > 128) return mvb::set_error(MVB_ERR_UNSUPPORTED, "codebook dim > 128");
  if (c->n_filters % c->compress) return mvb::set_error(MVB_ERR_UNSUPPORTED, "n_filters not a multiple of compress");
  const int top = c->n_filters << c->n_ratios;
  if (top < 32 || top % 32 || lstm_smem(top, 1) > (size_t)LSTM_SMEM_LIMIT)
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "LSTM width %d unsupported", top);
  for (int i = 0; i < c->n_ratios; ++i) {
    const int r = c->ratios[i];
    if (r != 2 && r != 4 && r != 5 && r != 8) return mvb::set_error(MVB_ERR_UNSUPPORTED, "downsampling ratio %d (2, 4, 5 or 8)", r);
  }
  if (c->kernel != 7 || c->res_kernel != 3 || c->last_kernel != 7) return mvb::set_error(MVB_ERR_UNSUPPORTED, "kernel sizes must be 7/3/7");
  if (c->max_frames < 1 || (long long)c->max_frames * enc_hop(c) > INT_MAX) return mvb::set_error(MVB_ERR_ARG, "max_frames out of range");
  return MVB_OK;
}

extern "C" size_t mvb_enc_workspace_bytes(const mvb_enc_config* c) {
  if (enc_validate(c)) return 0;
  return enc_layout(c, 1, c->max_frames).total + ENC_BOOKS_BYTES + enc_norms_bytes(c);
}

extern "C" int mvb_enc_create(const mvb_enc_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets, void* d_ws,
                              mvb_enc** out) {
  if (int e = enc_validate(cfg)) return e;
  if (!d_arena || !offsets || !d_ws || !out) return mvb::set_error(MVB_ERR_ARG, "null pointer argument");
  if (int e = check_offsets(offsets, enc_n_tensors(cfg), arena_bytes, "encoder: weight offset")) return e;
  if (int e = lstm_check_coresident(cfg->n_filters << cfg->n_ratios, 1)) return e;
  Building<mvb_enc> hb(new mvb_enc(), mvb_enc_destroy);
  mvb_enc* h = hb.get();
  h->cfg = *cfg;
  h->hop = enc_hop(cfg);
  h->arena = reinterpret_cast<const char*>(d_arena);
  h->off.assign(offsets, offsets + enc_n_tensors(cfg));
  const EncLayout L = enc_layout(cfg, 1, cfg->max_frames);
  h->bufs = enc_bufs(d_ws, L);
  h->books_dev = (const float**)(reinterpret_cast<char*>(d_ws) + L.total);
  h->norms = reinterpret_cast<float*>(reinterpret_cast<char*>(d_ws) + L.total + ENC_BOOKS_BYTES);
  std::vector<const float*> books(cfg->n_q);
  for (int q = 0; q < cfg->n_q; ++q) books[q] = h->w(q);
  MVB_CK(cudaMemcpy(h->books_dev, books.data(), sizeof(void*) * cfg->n_q, cudaMemcpyHostToDevice));
  k_sq_norms<<<dim3(ENC_BINS / 256, cfg->n_q), 256>>>(h->books_dev, cfg->hidden, h->norms);
  MVB_CK(cudaGetLastError());
  MVB_CK(cudaDeviceSynchronize());
  *out = hb.release();
  return MVB_OK;
}

extern "C" int mvb_enc_destroy(mvb_enc* h) {
  delete h;
  return MVB_OK;
}

static cudaError_t conv_down(cudaStream_t s, const float* x, int Cin, const Segs& segs, int n, int T_max, int m, int S,
                             const float* w, const float* b, float* y, int Cout) {
  const dim3 grid((T_max * m / S + 255) / 256, (Cout + 31) / 32, n);
  switch (S) {
    case 2: k_conv1d_down<2><<<grid, 256, 0, s>>>(x, Cin, segs, m, w, b, y, Cout); break;
    case 4: k_conv1d_down<4><<<grid, 256, 0, s>>>(x, Cin, segs, m, w, b, y, Cout); break;
    case 5: k_conv1d_down<5><<<grid, 256, 0, s>>>(x, Cin, segs, m, w, b, y, Cout); break;
    case 8: k_conv1d_down<8><<<grid, 256, 0, s>>>(x, Cin, segs, m, w, b, y, Cout); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

static cudaError_t rvq_encode(cudaStream_t s, const float* emb, int dim, const Segs& segs, int n, int T_max, const float* const* books,
                              const float* norms, int n_q, int32_t* codes, float* res_out) {
  k_rvq_encode<<<dim3((T_max + 31) / 32, 1, n), 256, 0, s>>>(emb, dim, segs, books, norms, n_q, codes, res_out);
  return cudaGetLastError();
}

// The segment list at m samples per frame: len_i = ceil(L_i m / hop).  L holds the input lengths.
static Segs at_rate(const Segs& frames, const int32_t* L, int n, int m, int hop) {
  Segs g = frames;
  for (int i = 0; i < n; ++i) g.s[i].len = (int)(((long long)L[i] * m + hop - 1) / hop);
  return g;
}

// The encoder's launch sequence over n validated utterances (frames: {F_i, off_i}, L: samples), one launch per layer for
// all of them.  The caller has checked that the LSTM is co-resident at n; b is a workspace laid out by enc_layout for at
// least n utterances and their frames.
static int enc_encode_segments(const mvb_enc* h, const float* d_wav, const Segs& frames, const int32_t* L, int n, int F_max,
                               const EncBufs& b, int32_t* d_codes, float* d_emb, cudaStream_t s) {
  const mvb_enc_config& c = h->cfg;
  const int hop = h->hop, top = c.n_filters << c.n_ratios;
  int L_max = 0;
  for (int i = 0; i < n; ++i) L_max = L[i] > L_max ? L[i] : L_max;
  int m = hop, ch = c.n_filters, ti = c.n_q;
  Segs g = at_rate(frames, L, n, m, hop);
  k_pack_wav<<<dim3((L_max + 255) / 256, 1, n), 256, 0, s>>>(d_wav, g, hop, b.B);
  MVB_CK(cudaGetLastError());
  MVB_CK(conv<7>(s, b.B, 1, g, n, F_max, m, h->w(ti), h->w(ti + 1), b.A, ch, 0, 0));            // conv_in
  ti += 2;
  for (int i = c.n_ratios - 1; i >= 0; --i) {
    const int r = c.ratios[i], hid = ch / c.compress;
    // resnet block: x = shortcut(u) + conv_k1(elu(conv_k3(elu(u))))  (u = A, result in C), then ELU + strided conv -> A
    MVB_CK(conv<3>(s, b.A, ch, g, n, F_max, m, h->w(ti), h->w(ti + 1), b.B, hid, 1, 0));
    MVB_CK(conv<1>(s, b.A, ch, g, n, F_max, m, h->w(ti + 4), h->w(ti + 5), b.C, ch, 0, 0));
    MVB_CK(conv<1>(s, b.B, hid, g, n, F_max, m, h->w(ti + 2), h->w(ti + 3), b.C, ch, 1, 1));
    MVB_CK(conv_down(s, b.C, ch, g, n, F_max, m, r, h->w(ti + 6), h->w(ti + 7), b.A, 2 * ch));
    m /= r;
    ch *= 2;
    ti += 8;
    g = at_rate(frames, L, n, m, hop);
  }
  // LSTM at one sample per frame (len_i = F_i): x = A;  layer 0 -> B ; layer 1 (+ skip x) -> C
  if (int e = lstm_set_smem_limit()) return e;
  const float* lin = b.A;
  float* louts[2] = {b.B, b.C};
  for (int l = 0; l < 2; ++l) {
    MVB_CK(conv<1>(s, lin, top, g, n, F_max, 1, h->w(ti), h->w(ti + 2), b.pre, 4 * top, 0, 0));     // W_ih x + (b_ih + b_hh)
    MVB_CK(lstm(s, b.pre, h->w(ti + 1), top, g, n, F_max, b.hbuf, b.bar, louts[l], l == 1 ? b.A : nullptr));
    lin = louts[l];
    ti += 3;
  }
  float* emb = d_emb ? d_emb : b.emb;
  MVB_CK(conv<7>(s, b.C, top, g, n, F_max, 1, h->w(ti), h->w(ti + 1), emb, c.hidden, 1, 0));     // ELU + conv_out
  MVB_CK(rvq_encode(s, emb, c.hidden, g, n, F_max, h->books_dev, h->norms, c.n_q, d_codes, nullptr));
  return MVB_OK;
}

static int enc_capacity(int max_batch, int max_total_frames) {
  if (max_batch < 1 || max_batch > CODEC_MAX_BATCH)
    return mvb::set_error(MVB_ERR_ARG, "encoder batch: max_batch %d out of range [1, %d]", max_batch, CODEC_MAX_BATCH);
  if (max_total_frames < 1) return mvb::set_error(MVB_ERR_ARG, "encoder batch: max_total_frames %d < 1", max_total_frames);
  return MVB_OK;
}

// Validates a batch (nothing is launched on failure) and builds its frame segment list; *F_max = the longest utterance.
static int enc_batch_segments(const mvb_enc* h, int n, const float* d_wav, const int32_t* L, int max_batch, int max_total_frames,
                              const int32_t* d_codes, Segs* segs, int* F_max) {
  if (!h || !d_wav || !L || !d_codes) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (int e = enc_capacity(max_batch, max_total_frames)) return e;
  if (n < 1 || n > max_batch) return mvb::set_error(MVB_ERR_ARG, "encoder batch: %d utterances, capacity %d", n, max_batch);
  const long long L_cap = (long long)h->hop * h->cfg.max_frames;
  *segs = Segs{};
  long long total = 0;
  int fmax = 0;
  for (int i = 0; i < n; ++i) {
    if (L[i] < 1 || L[i] > L_cap)
      return mvb::set_error(MVB_ERR_ARG, "encoder batch: utterance %d: %d samples out of range [1, %lld]", i, L[i], L_cap);
    const int F = (L[i] + h->hop - 1) / h->hop;
    segs->s[i] = Seg{F, (int)total, F};
    total += F;
    if (F > fmax) fmax = F;
  }
  if (total > max_total_frames)
    return mvb::set_error(MVB_ERR_ARG, "encoder batch: %lld frames in all, capacity %d", total, max_total_frames);
  *F_max = fmax;
  return MVB_OK;
}

extern "C" int mvb_enc_encode(mvb_enc* h, const float* d_wav, int32_t L, int32_t* d_codes, float* d_emb, void* stream) {
  Segs segs;
  int F_max = 0;
  if (int e = enc_batch_segments(h, 1, d_wav, &L, 1, h ? h->cfg.max_frames : 1, d_codes, &segs, &F_max)) return e;
  return enc_encode_segments(h, d_wav, segs, &L, 1, F_max, h->bufs, d_codes, d_emb, (cudaStream_t)stream);
}

extern "C" size_t mvb_enc_batch_workspace_bytes(const mvb_enc_config* c, int32_t max_batch, int32_t max_total_frames) {
  if (enc_validate(c) || enc_capacity(max_batch, max_total_frames)) return 0;
  return enc_layout(c, max_batch, max_total_frames).total;
}

extern "C" int mvb_enc_encode_batch(mvb_enc* h, int32_t n, const float* d_wav, const int32_t* L, void* d_batch_ws, int32_t max_batch,
                                    int32_t max_total_frames, int32_t* d_codes, float* d_emb, void* stream) {
  Segs segs;
  int F_max = 0;
  if (!d_batch_ws) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (int e = enc_batch_segments(h, n, d_wav, L, max_batch, max_total_frames, d_codes, &segs, &F_max)) return e;
  if (int e = lstm_check_coresident(h->cfg.n_filters << h->cfg.n_ratios, n)) return e;
  const EncBufs b = enc_bufs(d_batch_ws, enc_layout(&h->cfg, max_batch, max_total_frames));
  return enc_encode_segments(h, d_wav, segs, L, n, F_max, b, d_codes, d_emb, (cudaStream_t)stream);
}

extern "C" int mvb_enc_op_test(int32_t op, const float* d_x, int32_t Cin, int32_t T, int32_t V, const float* d_w, const float* d_b,
                               int32_t Cout, int32_t k, int32_t elu_in, float* d_y, int32_t* d_codes, void* stream) {
  if (!d_x || !d_w) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (Cin < 1 || T < 1 || V < 1 || V > T) return mvb::set_error(MVB_ERR_ARG, "mvb_enc_op_test: bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  const Segs one = one_segment(T, V);
  if (op == 0) {
    if (Cout < 1 || !d_b || !d_y) return mvb::set_error(MVB_ERR_ARG, "mvb_enc_op_test: bad shape or null bias / output");
    if (k != 2 && k != 4 && k != 5 && k != 8) return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_enc_op_test: stride %d", k);
    if (T % k) return mvb::set_error(MVB_ERR_ARG, "mvb_enc_op_test: T %% stride != 0");
    MVB_CK(conv_down(s, d_x, Cin, one, 1, T, 1, k, d_w, d_b, d_y, Cout));
  } else if (op == 1) {
    if (Cout < 1 || !d_y) return mvb::set_error(MVB_ERR_ARG, "mvb_enc_op_test: bad shape or null output");
    if (k == 1) MVB_CK(conv<1>(s, d_x, Cin, one, 1, T, 1, d_w, d_b, d_y, Cout, elu_in, 0));
    else if (k == 3) MVB_CK(conv<3>(s, d_x, Cin, one, 1, T, 1, d_w, d_b, d_y, Cout, elu_in, 0));
    else if (k == 7) MVB_CK(conv<7>(s, d_x, Cin, one, 1, T, 1, d_w, d_b, d_y, Cout, elu_in, 0));
    else return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_enc_op_test: conv kernel size %d", k);
  } else if (op == 2) {
    const int dim = Cin, n_q = k;
    if (dim > 128 || n_q < 1 || n_q > 64 || !d_codes) return mvb::set_error(MVB_ERR_ARG, "mvb_enc_op_test: bad RVQ shape");
    WsBump ws;
    const size_t o_tab = ws.take(sizeof(void*) * n_q), o_nrm = ws.take((size_t)n_q * ENC_BINS * 4);
    char* buf = nullptr;
    MVB_CK(cudaMalloc(&buf, ws.end));
    std::vector<const float*> books(n_q);
    for (int q = 0; q < n_q; ++q) books[q] = d_w + (size_t)q * ENC_BINS * dim;
    const float** tab = reinterpret_cast<const float**>(buf + o_tab);
    float* nrm = reinterpret_cast<float*>(buf + o_nrm);
    const Segs frames = one_segment(T, T);
    cudaError_t e = cudaMemcpyAsync(tab, books.data(), sizeof(void*) * n_q, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
      k_sq_norms<<<dim3(ENC_BINS / 256, n_q), 256, 0, s>>>(tab, dim, nrm);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = rvq_encode(s, d_x, dim, frames, 1, T, tab, nrm, n_q, d_codes, d_y);
    const cudaError_t es = cudaStreamSynchronize(s);   // (also on an error path: the buffer is freed only once unused)
    cudaFree(buf);
    if (e == cudaSuccess) e = es;
    if (e != cudaSuccess) return mvb::set_error(MVB_ERR_CUDA, "mvb_enc_op_test: %s", cudaGetErrorString(e));
    return MVB_OK;
  } else {
    return mvb::set_error(MVB_ERR_ARG, "mvb_enc_op_test: op %d", op);
  }
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}
