// EnCodec-24 kHz decode path of the vocoder (SURVEY.md row a17, first half): RVQ decode -> SEANet decoder.
// This is what `mbd.tokens_to_wav` (fam/llm/decoders.py:85 -> audiocraft 1.2.0) computes first, as the loudness /
// band-energy reference and as the diffusion condition (`decode_latent`).  audiocraft delegates the 24 kHz codec to
// transformers.EncodecModel; operator semantics follow modeling_encodec.py (cited per kernel).  fp32 throughout
// (the reference forces fp32 autocast for the vocoder, decoders.py:84).
//
// Activations are [C][T] fp32 per utterance (time contiguous): every conv streams its input window through a
// shared-memory line buffer (128-bit coalesced loads of the tile body, scalar loads for the K-1 halo samples), keeps an
// 8-channel x 4-sample register tile per thread and writes it back with 128-bit stores.
//
// Every kernel decodes n <= 32 utterances in one launch over the segment list of codec.cuh (k_conv1d and k_lstm_layer
// live there: the encoder runs them too).  Decoder blocks are full (len = SEG_WHOLE).  A single-utterance decode is the
// list {T, 0}.
#include <cuda_runtime.h>

#include <vector>

#include "codec.cuh"
#include "common.cuh"
#include "host.cuh"

using namespace mvb;

namespace {

// latent[c][t] = sum_q codebook_q[codes[q][t]][c]     (EncodecResidualVectorQuantizer.decode)
// One tile of 32 frames: codes [n_q, T] at n_q off -> out [dim, T] at dim off.
__global__ void __launch_bounds__(128) k_rvq_decode(const int* __restrict__ codes, int n_q, Segs segs,
                                                    const float* const* __restrict__ books, int dim, float* __restrict__ out) {
  __shared__ float tile[32][129];
  const Seg g = segs.s[blockIdx.z];
  const int T = g.T, t0 = blockIdx.x * 32;
  if (t0 >= T) return;
  codes += (size_t)n_q * g.off;
  out += (size_t)dim * g.off;
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

// ConvTranspose1d(k = 2r, stride r) trimmed by r samples on the right (EncodecConvTranspose1d, causal) with the
// preceding ELU fused:  y[co][t*r + p] = b[co] + sum_ci w[ci][co][p] * e[ci][t] + w[ci][co][p + r] * e[ci][t-1].
// Input at m samples per frame, output at m r: x [Cin, T] -> y [Cout, T r] per utterance; one tile = 32 input samples.
__global__ void __launch_bounds__(256) k_convtr1d(const float* __restrict__ x, int Cin, Segs segs, int m, const float* __restrict__ w,
                                                  const float* __restrict__ bias, float* __restrict__ y, int Cout, int r) {
  constexpr int CI = 16, TI = 32, CO = 32;
  extern __shared__ float sm[];
  float* xs = sm;                       // [CI][TI + 1]   (index 0 = t0 - 1)
  float* ws = sm + CI * (TI + 1);       // [CI][CO][2r]
  // The segment goes through shared memory: read from the parameter directly, its fields stay in uniform registers and
  // ptxas, at 64 registers, recomputes the inner loop's addresses (7 % slower on an H100) or spills.
  __shared__ Seg gs;
  if (threadIdx.x == 0) gs = segs.s[blockIdx.z];
  __syncthreads();
  const Seg g = gs;
  const int T = g.T * m, t0 = blockIdx.x * TI, co0 = blockIdx.y * CO;
  if (t0 >= T) return;
  const float* __restrict__ xb = x + (size_t)g.off * m * Cin;
  float* __restrict__ yb = y + (size_t)g.off * m * r * Cout;
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

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// Decoder workspace for max_batch utterances of max_total_frames frames in all: three activation buffers | LSTM
// pre-activations | h exchange [2][max_batch][H] | barrier word.  A batch workspace is this layout; the handle's own
// workspace is this layout at (1, max_frames) followed by the codebook pointer table.
struct VocLayout { size_t A, B, C, pre, h, bar, total; };
struct VocBufs { float *A, *B, *C, *pre, *hbuf; unsigned* bar; };

struct mvb_voc {
  mvb_voc_config cfg;
  const char* arena;
  std::vector<uint64_t> off;
  VocBufs bufs;                 // in the handle's workspace: single-utterance decodes
  const float** books_dev;
  const float* w(int i) const { return reinterpret_cast<const float*>(arena + off[i]); }
};

// tensor order in the arena (fp32, weight norm folded by the loader):
//   codebooks[n_q] | conv_in {w,b} | lstm l0 {w_ih, w_hh, b_ih+b_hh} | lstm l1 {...} |
//   per ratio: up {w,b}, res.c1 {w,b}, res.c2 {w,b}, res.shortcut {w,b} | conv_out {w,b}
static int voc_n_tensors(const mvb_voc_config* c) { return c->n_q + 2 + 6 + c->n_ratios * 8 + 2; }

static VocLayout voc_layout(const mvb_voc_config* c, int max_batch, int max_total_frames) {
  const size_t T = (size_t)max_total_frames;
  // elements of the largest activation (channels x samples, over the upsampling stages)
  int ch = c->n_filters << c->n_ratios;   // 512
  size_t maxelems = (size_t)ch * T, Tl = T;
  for (int i = 0; i < c->n_ratios; ++i) {
    Tl *= c->ratios[i];
    ch >>= 1;
    if ((size_t)ch * Tl > maxelems) maxelems = (size_t)ch * Tl;
  }
  const size_t top = (size_t)(c->n_filters << c->n_ratios);
  VocLayout L;
  WsBump ws;
  L.A = ws.take(maxelems * 4); L.B = ws.take(maxelems * 4); L.C = ws.take(maxelems * 4);
  L.pre = ws.take(4 * top * T * 4);
  L.h = ws.take(2 * (size_t)max_batch * top * 4);
  L.bar = ws.take(256);
  L.total = ws.end;
  return L;
}

static VocBufs voc_bufs(void* d_ws, const VocLayout& L) {
  char* ws = reinterpret_cast<char*>(d_ws);
  return VocBufs{(float*)(ws + L.A), (float*)(ws + L.B), (float*)(ws + L.C), (float*)(ws + L.pre), (float*)(ws + L.h),
                 (unsigned*)(ws + L.bar)};
}

constexpr size_t VOC_BOOKS_BYTES = 64 * sizeof(void*);   // codebook pointer table, after voc_layout(1, max_frames)

static int voc_validate(const mvb_voc_config* c) {
  if (!c) return mvb::set_error(MVB_ERR_ARG, "null config");
  if (c->n_ratios < 1 || c->n_ratios > 8 || c->n_q < 1 || c->n_q > 32) return mvb::set_error(MVB_ERR_ARG, "bad codec shape");
  if (c->hidden > 128) return mvb::set_error(MVB_ERR_UNSUPPORTED, "codebook dim > 128");
  const int top = c->n_filters << c->n_ratios;
  if (top < 32 || top % 32 || lstm_smem(top, 1) > (size_t)LSTM_SMEM_LIMIT)
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "LSTM width %d unsupported", top);
  for (int i = 0; i < c->n_ratios; ++i)
    if (c->ratios[i] < 1 || c->ratios[i] > 8) return mvb::set_error(MVB_ERR_UNSUPPORTED, "upsampling ratio out of range");
  if (c->kernel != 7 || c->res_kernel != 3 || c->last_kernel != 7) return mvb::set_error(MVB_ERR_UNSUPPORTED, "kernel sizes must be 7/3/7");
  if (c->max_frames < 8) return mvb::set_error(MVB_ERR_ARG, "max_frames too small");
  return MVB_OK;
}

extern "C" size_t mvb_voc_workspace_bytes(const mvb_voc_config* c) {
  if (voc_validate(c)) return 0;
  return voc_layout(c, 1, c->max_frames).total + VOC_BOOKS_BYTES;
}

extern "C" int mvb_voc_create(const mvb_voc_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets, void* d_ws,
                              mvb_voc** out) {
  if (int e = voc_validate(cfg)) return e;
  if (!d_arena || !offsets || !d_ws || !out) return mvb::set_error(MVB_ERR_ARG, "null pointer argument");
  if (int e = check_offsets(offsets, voc_n_tensors(cfg), arena_bytes, "vocoder: weight offset")) return e;
  if (int e = lstm_check_coresident(cfg->n_filters << cfg->n_ratios, 1)) return e;
  Building<mvb_voc> hb(new mvb_voc(), mvb_voc_destroy);
  mvb_voc* h = hb.get();
  h->cfg = *cfg;
  h->arena = reinterpret_cast<const char*>(d_arena);
  h->off.assign(offsets, offsets + voc_n_tensors(cfg));
  const VocLayout L = voc_layout(cfg, 1, cfg->max_frames);
  h->bufs = voc_bufs(d_ws, L);
  h->books_dev = (const float**)(reinterpret_cast<char*>(d_ws) + L.total);
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

static cudaError_t convtr(cudaStream_t s, const float* x, int Cin, const Segs& segs, int n, int T_max, int m, const float* w,
                          const float* b, float* y, int Cout, int r) {
  const size_t smem = (size_t)(16 * 33 + 16 * 32 * 2 * r) * 4;
  k_convtr1d<<<dim3((T_max * m + 31) / 32, (Cout + 31) / 32, n), 256, smem, s>>>(x, Cin, segs, m, w, b, y, Cout, r);
  return cudaGetLastError();
}

// RVQ decode of n validated segments: codes -> d_latent.
static int voc_latent_segments(const mvb_voc* h, const int32_t* d_codes, const Segs& segs, int n, int T_max, float* d_latent,
                               cudaStream_t s) {
  k_rvq_decode<<<dim3((T_max + 31) / 32, 1, n), 128, 0, s>>>(d_codes, h->cfg.n_q, segs, h->books_dev, h->cfg.hidden, d_latent);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

// The decoder's launch sequence over n validated segments, one launch per layer for all of them: codes -> d_wav.  The
// caller has checked that the LSTM is co-resident at n; b is a workspace laid out by voc_layout for at least n utterances
// and their frames.
static int voc_decode_segments(const mvb_voc* h, const int32_t* d_codes, const Segs& segs, int n, int T_max, const VocBufs& b,
                               float* d_wav, cudaStream_t s) {
  const mvb_voc_config& c = h->cfg;
  const int top = c.n_filters << c.n_ratios;
  int ti = c.n_q;
  if (int e = voc_latent_segments(h, d_codes, segs, n, T_max, b.A, s)) return e;
  MVB_CK(conv<7>(s, b.A, c.hidden, segs, n, T_max, 1, h->w(ti), h->w(ti + 1), b.B, top, 0, 0));      // conv_in
  ti += 2;
  // LSTM: x = B;  layer 0 -> A ; layer 1 (+ skip x) -> C
  if (int e = lstm_set_smem_limit()) return e;
  const float* lin = b.B;
  float* louts[2] = {b.A, b.C};
  for (int l = 0; l < 2; ++l) {
    MVB_CK(conv<1>(s, lin, top, segs, n, T_max, 1, h->w(ti), h->w(ti + 2), b.pre, 4 * top, 0, 0));   // W_ih x + (b_ih + b_hh)
    MVB_CK(lstm(s, b.pre, h->w(ti + 1), top, segs, n, T_max, b.hbuf, b.bar, louts[l], l == 1 ? b.B : nullptr));
    lin = louts[l];
    ti += 3;
  }
  float* x = b.C;          // current activation
  float* f1 = b.A;
  float* f2 = b.B;
  int ch = top, m = 1;
  for (int i = 0; i < c.n_ratios; ++i) {
    const int r = c.ratios[i], co = ch / 2;
    MVB_CK(convtr(s, x, ch, segs, n, T_max, m, h->w(ti), h->w(ti + 1), f1, co, r));
    m *= r; ch = co;
    // resnet block: y = shortcut(u) + conv_k1(elu(conv_k3(elu(u))))
    MVB_CK(conv<3>(s, f1, ch, segs, n, T_max, m, h->w(ti + 2), h->w(ti + 3), f2, ch / c.compress, 1, 0));
    MVB_CK(conv<1>(s, f1, ch, segs, n, T_max, m, h->w(ti + 6), h->w(ti + 7), x, ch, 0, 0));
    MVB_CK(conv<1>(s, f2, ch / c.compress, segs, n, T_max, m, h->w(ti + 4), h->w(ti + 5), x, ch, 1, 1));
    ti += 8;
  }
  MVB_CK(conv<7>(s, x, ch, segs, n, T_max, m, h->w(ti), h->w(ti + 1), d_wav, 1, 1, 0));
  return MVB_OK;
}

// RVQ decode only: the diffusion condition `decode_latent` (and the decoder's input).  d_codes int32 [n_q, T].
extern "C" int mvb_voc_decode_latent(mvb_voc* h, const int32_t* d_codes, int32_t T, float* d_latent, void* stream) {
  if (!h || !d_codes || !d_latent) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (T < 1 || T > h->cfg.max_frames) return mvb::set_error(MVB_ERR_ARG, "frame count %d out of range", T);
  return voc_latent_segments(h, d_codes, one_segment(T), 1, T, d_latent, (cudaStream_t)stream);
}

// codes int32 [n_q, T] -> waveform fp32 [T * prod(ratios)]   (== EncodecModel.decode for one chunk)
extern "C" int mvb_voc_decode(mvb_voc* h, const int32_t* d_codes, int32_t T, float* d_wav, void* stream) {
  if (!h || !d_codes || !d_wav) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (T < 8 || T > h->cfg.max_frames) return mvb::set_error(MVB_ERR_ARG, "frame count %d out of range [8, %d]", T, h->cfg.max_frames);
  return voc_decode_segments(h, d_codes, one_segment(T), 1, T, h->bufs, d_wav, (cudaStream_t)stream);
}

// ---- batched decode: a caller-owned workspace of voc_layout(max_batch, max_total_frames) -------------------------------
static int voc_batch_capacity(int max_batch, int max_total_frames) {
  if (max_batch < 1 || max_batch > CODEC_MAX_BATCH)
    return mvb::set_error(MVB_ERR_ARG, "vocoder batch: max_batch %d out of range [1, %d]", max_batch, CODEC_MAX_BATCH);
  if (max_total_frames < 8) return mvb::set_error(MVB_ERR_ARG, "vocoder batch: max_total_frames %d < 8", max_total_frames);
  return MVB_OK;
}

extern "C" size_t mvb_voc_batch_workspace_bytes(const mvb_voc_config* c, int32_t max_batch, int32_t max_total_frames) {
  if (voc_validate(c) || voc_batch_capacity(max_batch, max_total_frames)) return 0;
  return voc_layout(c, max_batch, max_total_frames).total;
}

// Validates a batch (nothing is launched on failure) and builds its segment list; *T_max = the longest utterance.
static int voc_batch_segments(const mvb_voc* h, int n, const int32_t* d_codes, const int32_t* T, const void* d_ws, int max_batch,
                              int max_total_frames, const void* d_out, Segs* segs, int* T_max) {
  if (!h || !d_codes || !T || !d_ws || !d_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (int e = voc_batch_capacity(max_batch, max_total_frames)) return e;
  if (n < 1 || n > max_batch) return mvb::set_error(MVB_ERR_ARG, "vocoder batch: %d utterances, capacity %d", n, max_batch);
  *segs = Segs{};
  long long total = 0;
  int tmax = 0;
  for (int i = 0; i < n; ++i) {
    if (T[i] < 8 || T[i] > h->cfg.max_frames)
      return mvb::set_error(MVB_ERR_ARG, "vocoder batch: utterance %d: frame count %d out of range [8, %d]", i, T[i], h->cfg.max_frames);
    segs->s[i] = Seg{T[i], (int)total, SEG_WHOLE};
    total += T[i];
    if (T[i] > tmax) tmax = T[i];
  }
  if (total > max_total_frames)
    return mvb::set_error(MVB_ERR_ARG, "vocoder batch: %lld frames in all, capacity %d", total, max_total_frames);
  *T_max = tmax;
  return MVB_OK;
}

extern "C" int mvb_voc_decode_latent_batch(mvb_voc* h, int32_t n, const int32_t* d_codes, const int32_t* T, void* d_batch_ws,
                                           int32_t max_batch, int32_t max_total_frames, float* d_latent, void* stream) {
  Segs segs;
  int T_max = 0;
  if (int e = voc_batch_segments(h, n, d_codes, T, d_batch_ws, max_batch, max_total_frames, d_latent, &segs, &T_max)) return e;
  return voc_latent_segments(h, d_codes, segs, n, T_max, d_latent, (cudaStream_t)stream);
}

extern "C" int mvb_voc_decode_batch(mvb_voc* h, int32_t n, const int32_t* d_codes, const int32_t* T, void* d_batch_ws,
                                    int32_t max_batch, int32_t max_total_frames, float* d_wav, void* stream) {
  Segs segs;
  int T_max = 0;
  if (int e = voc_batch_segments(h, n, d_codes, T, d_batch_ws, max_batch, max_total_frames, d_wav, &segs, &T_max)) return e;
  if (int e = lstm_check_coresident(h->cfg.n_filters << h->cfg.n_ratios, n)) return e;
  const VocBufs b = voc_bufs(d_batch_ws, voc_layout(&h->cfg, max_batch, max_total_frames));
  return voc_decode_segments(h, d_codes, segs, n, T_max, b, d_wav, (cudaStream_t)stream);
}

extern "C" int mvb_voc_op_test(int32_t op, const float* d_x, int32_t Cin, int32_t T, const float* d_w, const float* d_b,
                               int32_t Cout, int32_t k, int32_t elu_in, int32_t accumulate, const float* d_skip, float* d_y,
                               void* stream) {
  if (!d_x || !d_w || !d_y) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (Cin < 1 || T < 1) return mvb::set_error(MVB_ERR_ARG, "mvb_voc_op_test: bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  const Segs one = one_segment(T);
  if (op == 0) {
    if (Cout < 1) return mvb::set_error(MVB_ERR_ARG, "mvb_voc_op_test: bad shape");
    if (k == 1) MVB_CK(conv<1>(s, d_x, Cin, one, 1, T, 1, d_w, d_b, d_y, Cout, elu_in, accumulate));
    else if (k == 3) MVB_CK(conv<3>(s, d_x, Cin, one, 1, T, 1, d_w, d_b, d_y, Cout, elu_in, accumulate));
    else if (k == 7) MVB_CK(conv<7>(s, d_x, Cin, one, 1, T, 1, d_w, d_b, d_y, Cout, elu_in, accumulate));
    else return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_voc_op_test: conv kernel size %d", k);
  } else if (op == 1) {
    if (Cout < 1 || !d_b) return mvb::set_error(MVB_ERR_ARG, "mvb_voc_op_test: bad shape or null bias");
    if (k < 1 || k > 8) return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_voc_op_test: upsampling ratio %d", k);
    MVB_CK(convtr(s, d_x, Cin, one, 1, T, 1, d_w, d_b, d_y, Cout, k));
  } else if (op == 2) {
    const int H = Cin;
    if (H % 32 || lstm_smem(H, 1) > (size_t)LSTM_SMEM_LIMIT) return mvb::set_error(MVB_ERR_UNSUPPORTED, "LSTM width %d unsupported", H);
    if (int e = lstm_check_coresident(H, 1)) return e;
    WsBump ws;
    const size_t o_h = ws.take((size_t)2 * H * 4), o_bar = ws.take(4);
    char* buf = nullptr;
    MVB_CK(cudaMalloc(&buf, ws.end));
    cudaError_t e = lstm(s, d_x, d_w, H, one, 1, T, reinterpret_cast<float*>(buf + o_h), reinterpret_cast<unsigned*>(buf + o_bar), d_y,
                         d_skip);
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
