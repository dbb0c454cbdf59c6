// Speaker encoder on the device (SURVEY.md row N3): 16 kHz waveform -> power mel spectrogram -> 3-layer LSTM over
// 160-frame partial windows -> linear -> ReLU -> L2 norm -> mean over the windows -> L2 norm.
//   fam/quantiser/audio/speaker_encoder/audio.py:10-22   wav_to_mel_spectrogram (librosa.feature.melspectrogram:
//                                                        centered STFT n_fft 400 / hop 160, periodic Hann, |X|^2,
//                                                        Slaney mel filterbank, 40 bands)
//   fam/quantiser/audio/speaker_encoder/model.py:50-53   forward
//   fam/quantiser/audio/speaker_encoder/model.py:81-103  embed_utterance (partial windows come from the host:
//                                                        compute_partial_slices is integer arithmetic, :55-79)
// fp32 throughout.  The job is latency-bound and tiny (1.4 M parameters, runs once per speaker): one CTA per partial
// window walks the 160 x 3 recurrent steps with the weights served from L2; one CTA per frame does the 400-point DFT.
#include <cuda_runtime.h>

#include <climits>
#include <cmath>
#include <algorithm>
#include <numeric>
#include <vector>

#include "common.cuh"
#include "host.cuh"

using namespace mvb;

namespace {

constexpr int SPK_THREADS = 256;

constexpr int SPK_MAX_BATCH = MVB_SPK_MAX_BATCH;

// Utterance i of a launch (blockIdx.z, or blockIdx.x for k_spk_mean): its n_wav samples at wav + wav_off, read as
// zero-extended to n_frames mel frames at mel frame mel_off; its n_part partial embeddings at row part_off.  The
// single-utterance entry points launch a list of one.
struct SpkSeg { long long wav_off; int n_wav, n_frames, mel_off, part_off, n_part; };
struct SpkSegs { SpkSeg s[SPK_MAX_BATCH]; };   // a kernel parameter (1 KB): indexing it needs no device table

// One frame per CTA: frame f covers samples [f*hop - n_fft/2, f*hop + n_fft/2) (center=True, zero padding).
__global__ void __launch_bounds__(SPK_THREADS) k_spk_mel(const float* __restrict__ wav, SpkSegs segs, int n_fft, int hop,
                                                         const float* __restrict__ window, const float* __restrict__ cosT,
                                                         const float* __restrict__ sinT, const float* __restrict__ melfb,
                                                         int n_mels, float* __restrict__ mel) {
  extern __shared__ float sm[];
  float* frame = sm;                 // [n_fft]
  float* power = sm + n_fft;         // [n_fft/2 + 1]
  const SpkSeg g = segs.s[blockIdx.z];
  const int f = blockIdx.x, tid = threadIdx.x;
  if (f >= g.n_frames) return;
  const float* x = wav + g.wav_off;
  const int n_bins = n_fft / 2 + 1;
  for (int n = tid; n < n_fft; n += SPK_THREADS) {
    const long long s = (long long)f * hop - n_fft / 2 + n;
    frame[n] = (s >= 0 && s < g.n_wav) ? x[s] * window[n] : 0.f;
  }
  __syncthreads();
  for (int k = tid; k < n_bins; k += SPK_THREADS) {
    float re = 0.f, im = 0.f;
    int ph = 0;                      // (k * n) mod n_fft
    for (int n = 0; n < n_fft; ++n) {
      const float v = frame[n];
      re = fmaf(v, cosT[ph], re);
      im = fmaf(v, sinT[ph], im);
      ph += k;
      if (ph >= n_fft) ph -= n_fft;
    }
    power[k] = re * re + im * im;
  }
  __syncthreads();
  float* out = mel + ((size_t)g.mel_off + f) * n_mels;
  for (int m = tid; m < n_mels; m += SPK_THREADS) {
    const float* fb = melfb + (size_t)m * n_bins;
    float acc = 0.f;
    for (int k = 0; k < n_bins; ++k) acc = fmaf(fb[k], power[k], acc);
    out[m] = acc;
  }
}

struct SpkW {
  const float* w_ih[3];
  const float* w_hh[3];
  const float* b[3];      // b_ih + b_hh
  const float* lw;
  const float* lb;
};

__device__ __forceinline__ float sigm(float v) { return 1.f / (1.f + expf(-v)); }

// One partial window per CTA: 160 steps x 3 layers (torch.nn.LSTM, gate order i, f, g, o), then linear + ReLU + L2 norm.
// trace (optional, tests only): [n_partials][T][3 layers][h, c][256], the state after every layer step.
__global__ void __launch_bounds__(SPK_THREADS) k_spk_lstm(const float* __restrict__ mel, const int* __restrict__ starts, int n_frames,
                                                          int T, int n_mels, SpkW W, float* __restrict__ partial_out,
                                                          float* __restrict__ trace) {
  constexpr int H = 256;
  __shared__ float xin[64];
  __shared__ float hs[3][H];
  __shared__ float gates[4 * H];
  __shared__ float red[8];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int p = blockIdx.x, f0 = starts[p];
  float c[3] = {0.f, 0.f, 0.f};
  for (int l = 0; l < 3; ++l) hs[l][tid] = 0.f;
  __syncthreads();
  for (int t = 0; t < T; ++t) {
    if (tid < n_mels) {
      const int f = f0 + t;
      xin[tid] = f < n_frames ? mel[(size_t)f * n_mels + tid] : 0.f;
    }
    __syncthreads();
    for (int l = 0; l < 3; ++l) {
      const int K = l == 0 ? n_mels : H;
      const float* in = l == 0 ? xin : hs[l - 1];
      const float* hp = hs[l];
      // 1024 gate rows over 8 warps, 4 rows in flight per warp (independent accumulators hide the L2 latency)
      for (int r0 = warp * 4; r0 < 4 * H; r0 += 32) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float* wi = W.w_ih[l] + (size_t)(r0 + q) * K;
          const float* wh = W.w_hh[l] + (size_t)(r0 + q) * H;
          for (int k = lane; k < K; k += 32) acc[q] = fmaf(__ldg(wi + k), in[k], acc[q]);
#pragma unroll
          for (int k = lane; k < H; k += 32) acc[q] = fmaf(__ldg(wh + k), hp[k], acc[q]);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float s = warp_sum(acc[q]);
          if (lane == 0) gates[r0 + q] = s + W.b[l][r0 + q];
        }
      }
      __syncthreads();
      const float ig = sigm(gates[tid]), fg = sigm(gates[H + tid]), gg = tanhf(gates[2 * H + tid]), og = sigm(gates[3 * H + tid]);
      c[l] = fg * c[l] + ig * gg;
      const float hn = og * tanhf(c[l]);
      __syncthreads();               // every warp has finished reading hs[l] / gates
      hs[l][tid] = hn;
      if (trace) {
        float* tr = trace + (((size_t)p * T + t) * 3 + l) * 2 * H;
        tr[tid] = hn;
        tr[H + tid] = c[l];
      }
      __syncthreads();
    }
  }
  // embeds_raw = relu(linear(hidden[-1])); embeds = embeds_raw / ||embeds_raw||   (model.py:51-53)
  float e = W.lb[tid];
  const float* lw = W.lw + (size_t)tid * H;
  for (int k = 0; k < H; ++k) e = fmaf(lw[k], hs[2][k], e);
  e = fmaxf(e, 0.f);
  float ss = warp_sum(e * e);
  if (lane == 0) red[warp] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < 8; ++i) tot += red[i];
  partial_out[(size_t)p * H + tid] = e / sqrtf(tot);
}

// raw = mean over the partial embeddings; embed = raw / ||raw||_2     (model.py:96-100).  One utterance per CTA:
// partials rows [part_off, part_off + n_part) -> out row blockIdx.x.
__global__ void __launch_bounds__(SPK_THREADS) k_spk_mean(const float* __restrict__ partials, SpkSegs segs, float* __restrict__ out) {
  __shared__ float red[8];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int P = segs.s[blockIdx.x].n_part;
  const float* x = partials + (size_t)segs.s[blockIdx.x].part_off * 256;
  float m = 0.f;
  for (int p = 0; p < P; ++p) m += x[(size_t)p * 256 + tid];
  m /= (float)P;
  float ss = warp_sum(m * m);
  if (lane == 0) red[warp] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < 8; ++i) tot += red[i];
  out[(size_t)blockIdx.x * 256 + tid] = m / sqrtf(tot);
}

// ---- batched front-end: resampling and silence trimming ---------------------------------------------------------------

// scipy.signal.resample_poly (signal.py, upfirdn with the filter centred): output j of a signal is
//   y[j] = sum_q taps[r][q] x[m - q],  t = j down + half_len,  r = t mod up,  m = t div up,
// over the q with 0 <= m - q < n_in (the zero extension at both ends contributes nothing), q ascending, one fmaf chain
// from 0.  taps is the filter in polyphase order [up][P].  One output per thread; the signal is blockIdx.z.
struct RsSeg { long long in_off, out_off; int n_in, n_out; };
struct RsSegs { RsSeg s[SPK_MAX_BATCH]; };

__global__ void __launch_bounds__(256) k_resample_poly(const float* __restrict__ x, RsSegs segs, int up, int down, int half_len,
                                                       const float* __restrict__ taps, int P, float* __restrict__ y) {
  const RsSeg g = segs.s[blockIdx.z];
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= g.n_out) return;
  const long long t = (long long)j * down + half_len, m = t / up;
  const float* h = taps + (size_t)(t - m * up) * P;
  const float* xs = x + g.in_off;
  const long long q0 = m >= g.n_in ? m - g.n_in + 1 : 0, q1 = m < P - 1 ? m : P - 1;
  float acc = 0.f;
  for (long long q = q0; q <= q1; ++q) acc = fmaf(__ldg(h + q), __ldg(xs + (m - q)), acc);
  y[g.out_off + j] = acc;
}

// librosa.effects.trim framing (trim_silence in speaker_encoder.py): frame f of a signal covers samples
// [f 512 - 1024, f 512 + 1024), zero padded; 1 + n / 512 frames.
constexpr int TRIM_FRAME = 2048, TRIM_HOP = 512;
struct TrimSeg { long long off; int n, frame_off; };
struct TrimSegs { TrimSeg s[SPK_MAX_BATCH]; };

// One warp per frame: lane l sums the squares of samples l, l + 32, ... of the frame (64-term fmaf chain from 0), then the
// warp_sum butterfly; rms = sqrtf(sum / 2048) -> rms[frame_off + f].
__global__ void __launch_bounds__(256) k_trim_rms(const float* __restrict__ wav, TrimSegs segs, float* __restrict__ rms) {
  const TrimSeg g = segs.s[blockIdx.z];
  const int f = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (f >= 1 + g.n / TRIM_HOP) return;                         // whole warps leave together
  const float* x = wav + g.off;
  const long long s0 = (long long)f * TRIM_HOP - TRIM_FRAME / 2;
  float acc = 0.f;
  for (int k = lane; k < TRIM_FRAME; k += 32) {
    const long long s = s0 + k;
    if (s >= 0 && s < g.n) acc = fmaf(x[s], x[s], acc);
  }
  const float ss = warp_sum(acc);
  if (lane == 0) rms[g.frame_off + f] = sqrtf(ss * (1.f / TRIM_FRAME));
}

// One CTA per signal (blockIdx.x): ref = the largest frame RMS; the kept span runs from the first to the last frame with
// 20 log10(max(rms, 1e-10) / ref) > -top_db, tested as fl(max(rms, 1e-10) / ref) > thr = fl(10^(-top_db / 20)) (an IEEE
// division and one fp32 threshold: no transcendental, so a ratio on the threshold compares as it does in float64)
// -> spans[i] = {first 512, min(n, (last + 1) 512)}; {0, 0} when ref is 0 or no frame is kept.
__global__ void __launch_bounds__(256) k_trim_span(const float* __restrict__ rms, TrimSegs segs, float thr, int* __restrict__ spans) {
  __shared__ float red[8];
  __shared__ int lo[8], hi[8];
  const TrimSeg g = segs.s[blockIdx.x];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, F = 1 + g.n / TRIM_HOP;
  const float* r = rms + g.frame_off;
  float m = 0.f;
  for (int f = tid; f < F; f += 256) m = fmaxf(m, r[f]);
  m = warp_max(m);
  if (lane == 0) red[warp] = m;
  __syncthreads();
  float ref = 0.f;
  for (int i = 0; i < 8; ++i) ref = fmaxf(ref, red[i]);
  int first = INT_MAX, last = -1;
  if (ref > 0.f)
    for (int f = tid; f < F; f += 256)
      if (fmaxf(r[f], 1e-10f) / ref > thr) { first = min(first, f); last = max(last, f); }
  for (int o = 16; o > 0; o >>= 1) {
    first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
    last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
  }
  if (lane == 0) { lo[warp] = first; hi[warp] = last; }
  __syncthreads();
  if (tid == 0) {
    for (int i = 0; i < 8; ++i) { first = min(first, lo[i]); last = max(last, hi[i]); }
    const bool keep = last >= 0;
    spans[2 * blockIdx.x] = keep ? first * TRIM_HOP : 0;
    spans[2 * blockIdx.x + 1] = keep ? (int)min((long long)g.n, (long long)(last + 1) * TRIM_HOP) : 0;
  }
}

}  // namespace

// Workspace: mel spectrogram of the longest input | <= 1024 partial starts | <= 1024 partial embeddings
struct SpkLayout { size_t starts, partials, total; };
static SpkLayout spk_layout(const mvb_spk_config* c) {
  WsBump ws;
  ws.take((size_t)(1 + c->max_samples / c->hop) * c->n_mels * 4);   // the mel spectrogram starts the workspace
  const size_t starts = ws.take(4096), partials = ws.take((size_t)1024 * 256 * 4);
  return {starts, partials, ws.end};
}

struct mvb_spk {
  mvb_spk_config cfg;
  const char* arena;
  std::vector<uint64_t> off;
  char* ws;
  SpkLayout L;
  const float* w(int i) const { return reinterpret_cast<const float*>(arena + off[i]); }
  float* mel() const { return reinterpret_cast<float*>(ws); }
  int* starts() const { return reinterpret_cast<int*>(ws + L.starts); }
  float* partials() const { return reinterpret_cast<float*>(ws + L.partials); }
};

static int spk_validate(const mvb_spk_config* c) {
  if (!c) return mvb::set_error(MVB_ERR_ARG, "null config");
  if (c->hidden != 256 || c->emb != 256 || c->n_layers != 3)
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "speaker encoder: hidden/embedding 256 and 3 layers are supported (model.py:14-18)");
  if (c->n_mels < 1 || c->n_mels > 64 || c->n_fft < 2 || c->n_fft > 2048 || c->hop < 1 || c->partial_frames < 1 || c->max_samples < 1)
    return mvb::set_error(MVB_ERR_ARG, "speaker encoder: bad front-end configuration");
  return MVB_OK;
}

extern "C" size_t mvb_spk_workspace_bytes(const mvb_spk_config* c) {
  if (spk_validate(c)) return 0;
  return spk_layout(c).total;
}

extern "C" int mvb_spk_create(const mvb_spk_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                              void* d_ws, mvb_spk** out) {
  if (int e = spk_validate(cfg)) return e;
  if (!d_arena || !offsets || !d_ws || !out) return mvb::set_error(MVB_ERR_ARG, "null pointer argument");
  if (int e = check_offsets(offsets, MVB_SPK_TENSORS, arena_bytes, "speaker encoder: tensor offset")) return e;
  Building<mvb_spk> hb(new mvb_spk(), mvb_spk_destroy);
  mvb_spk* h = hb.get();
  h->cfg = *cfg;
  h->arena = reinterpret_cast<const char*>(d_arena);
  h->off.assign(offsets, offsets + MVB_SPK_TENSORS);
  h->ws = reinterpret_cast<char*>(d_ws);
  h->L = spk_layout(cfg);
  *out = hb.release();
  return MVB_OK;
}

extern "C" int mvb_spk_destroy(mvb_spk* h) {
  delete h;
  return MVB_OK;
}

// k_spk_mel over n utterances (segs: wav_off, n_wav, n_frames, mel_off); F_max = the most frames of one.
static int spk_mel_segments(const mvb_spk* h, const float* d_wav, const SpkSegs& segs, int n, int F_max, float* d_mel, cudaStream_t s) {
  const mvb_spk_config& c = h->cfg;
  const size_t smem = (size_t)(c.n_fft + c.n_fft / 2 + 1) * 4;
  // tensors: 3 x {w_ih, w_hh, b}, linear w, linear b, mel filterbank, window, cos table, sin table
  k_spk_mel<<<dim3(F_max, 1, n), SPK_THREADS, smem, s>>>(d_wav, segs, c.n_fft, c.hop, h->w(12), h->w(13), h->w(14), h->w(11), c.n_mels, d_mel);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

static int spk_mel(mvb_spk* h, const float* d_wav, int n_samples, float* d_mel, cudaStream_t s) {
  const int n_frames = 1 + n_samples / h->cfg.hop;
  SpkSegs segs{};
  segs.s[0] = SpkSeg{0, n_samples, n_frames, 0, 0, 0};
  return spk_mel_segments(h, d_wav, segs, 1, n_frames, d_mel, s);
}

extern "C" int mvb_spk_mel(mvb_spk* h, const float* d_wav, int32_t n_samples, float* d_mel, void* stream) {
  if (!h || !d_wav || !d_mel) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (n_samples < 1 || n_samples > h->cfg.max_samples) return mvb::set_error(MVB_ERR_ARG, "n_samples %d out of range", n_samples);
  return spk_mel(h, d_wav, n_samples, d_mel, (cudaStream_t)stream);
}

// The windows and the average, for mvb_spk_embed and mvb_spk_op_test alike.  With `starts` (HOST int32 [n_partials]):
// k_spk_lstm over the windows of d_mel [n_frames, n_mels] -> d_partials [n_partials, 256] (+ d_trace when non-null);
// with d_embed: k_spk_mean over d_partials -> d_embed [256].  Every window must lie inside the mel: k_spk_lstm reads frames
// start .. start + partial_frames - 1, and a window past either end is neither in the spectrogram nor a window the
// reference can form.
static int spk_check_windows(const mvb_spk* h, int n_frames, const int32_t* starts, int n_partials) {
  if (n_partials < 1 || n_partials > 1024) return mvb::set_error(MVB_ERR_ARG, "n_partials %d out of range", n_partials);
  if (!starts) return MVB_OK;
  for (int i = 0; i < n_partials; ++i)
    if (starts[i] < 0 || (long long)starts[i] + h->cfg.partial_frames > n_frames)
      return mvb::set_error(MVB_ERR_ARG, "window %d starts at mel frame %d: %d frames from there do not fit in %d", i, starts[i],
                            h->cfg.partial_frames, n_frames);
  return MVB_OK;
}

// k_spk_lstm over n_windows windows whose first frames (device int32) index d_mel [n_frames, n_mels].
static int spk_lstm(const mvb_spk* h, const float* d_mel, const int* d_starts, int n_frames, int n_windows, float* d_partials,
                    float* d_trace, cudaStream_t s) {
  const mvb_spk_config& c = h->cfg;
  SpkW W;
  for (int l = 0; l < 3; ++l) { W.w_ih[l] = h->w(3 * l); W.w_hh[l] = h->w(3 * l + 1); W.b[l] = h->w(3 * l + 2); }
  W.lw = h->w(9); W.lb = h->w(10);
  k_spk_lstm<<<n_windows, SPK_THREADS, 0, s>>>(d_mel, d_starts, n_frames, c.partial_frames, c.n_mels, W, d_partials, d_trace);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

static int spk_mean(const float* d_partials, const SpkSegs& segs, int n, float* d_embed, cudaStream_t s) {
  k_spk_mean<<<n, SPK_THREADS, 0, s>>>(d_partials, segs, d_embed);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

static int spk_windows(mvb_spk* h, const float* d_mel, int n_frames, const int32_t* starts, int n_partials, float* d_partials,
                       float* d_trace, float* d_embed, cudaStream_t s) {
  if (int e = spk_check_windows(h, n_frames, starts, n_partials)) return e;
  if (starts) {
    MVB_CK(cudaMemcpyAsync(h->starts(), starts, sizeof(int) * n_partials, cudaMemcpyHostToDevice, s));
    if (int e = spk_lstm(h, d_mel, h->starts(), n_frames, n_partials, d_partials, d_trace, s)) return e;
  }
  if (d_embed) {
    SpkSegs segs{};
    segs.s[0].n_part = n_partials;
    if (int e = spk_mean(d_partials, segs, 1, d_embed, s)) return e;
  }
  return MVB_OK;
}

extern "C" int mvb_spk_embed(mvb_spk* h, const float* d_wav, int32_t n_samples, const int32_t* slice_starts, int32_t n_partials,
                             float* d_embed, float* d_partials_out, void* stream) {
  if (!h || !d_wav || !slice_starts || !d_embed) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (n_samples < 1 || n_samples > h->cfg.max_samples) return mvb::set_error(MVB_ERR_ARG, "n_samples %d out of range", n_samples);
  cudaStream_t s = (cudaStream_t)stream;
  const int n_frames = 1 + n_samples / h->cfg.hop;
  if (int e = spk_check_windows(h, n_frames, slice_starts, n_partials)) return e;   // before anything is launched
  if (int e = spk_mel(h, d_wav, n_samples, h->mel(), s)) return e;
  if (int e = spk_windows(h, h->mel(), n_frames, slice_starts, n_partials, h->partials(), nullptr, d_embed, s)) return e;
  if (d_partials_out)
    MVB_CK(cudaMemcpyAsync(d_partials_out, h->partials(), sizeof(float) * (size_t)n_partials * 256, cudaMemcpyDeviceToDevice, s));
  return MVB_OK;
}

extern "C" int mvb_spk_op_test(mvb_spk* h, int32_t op, const float* d_in, int32_t n_frames, const int32_t* starts, int32_t n_partials,
                               float* d_out, float* d_trace, void* stream) {
  if (!h || !d_in || !d_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  int e;
  if (op == 0) {
    if (!starts) return mvb::set_error(MVB_ERR_ARG, "null argument");
    if (n_frames < 1) return mvb::set_error(MVB_ERR_ARG, "mvb_spk_op_test: n_frames %d", n_frames);
    e = spk_windows(h, d_in, n_frames, starts, n_partials, d_out, d_trace, nullptr, s);
  } else if (op == 1) {
    e = spk_windows(h, nullptr, 0, nullptr, n_partials, const_cast<float*>(d_in), nullptr, d_out, s);
  } else {
    return mvb::set_error(MVB_ERR_ARG, "mvb_spk_op_test: op %d", op);
  }
  if (e) return e;
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}

// ---- batched front-end -------------------------------------------------------------------------------------------------

extern "C" int mvb_resample_batch(int32_t n, const float* d_in, const int32_t* n_in, int32_t up, int32_t down, const float* d_taps,
                                  int32_t n_taps, float* d_out, void* stream) {
  if (!d_in || !n_in || !d_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (n < 1 || n > SPK_MAX_BATCH) return mvb::set_error(MVB_ERR_ARG, "resample: %d signals, 1 .. %d per call", n, SPK_MAX_BATCH);
  if (up < 1 || down < 1) return mvb::set_error(MVB_ERR_ARG, "resample: up %d / down %d", up, down);
  const int g = std::gcd(up, down);
  up /= g;
  down /= g;
  const long long want = 20LL * (up > down ? up : down) + 1;
  if (up != down) {
    if (want > MVB_RESAMPLE_MAX_TAPS)
      return mvb::set_error(MVB_ERR_UNSUPPORTED, "resample: %d/%d needs a %lld-tap filter, more than %d", up, down, want,
                            MVB_RESAMPLE_MAX_TAPS);
    if (!d_taps || n_taps != want) return mvb::set_error(MVB_ERR_ARG, "resample: %d/%d takes %lld taps, not %d", up, down, want, n_taps);
  }
  RsSegs segs{};
  long long in = 0, out = 0;
  int o_max = 0;
  for (int i = 0; i < n; ++i) {
    const long long o = ((long long)n_in[i] * up + down - 1) / down;
    if (n_in[i] < 1 || o > INT_MAX) return mvb::set_error(MVB_ERR_ARG, "resample: signal %d: %d samples", i, n_in[i]);
    segs.s[i] = RsSeg{in, out, n_in[i], (int)o};
    in += n_in[i];
    out += o;
    if (o > o_max) o_max = (int)o;
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (up == down) {
    MVB_CK(cudaMemcpyAsync(d_out, d_in, sizeof(float) * in, cudaMemcpyDeviceToDevice, s));
    return MVB_OK;
  }
  const int P = (int)((want + up - 1) / up);
  k_resample_poly<<<dim3((o_max + 255) / 256, 1, n), 256, 0, s>>>(d_in, segs, up, down, (int)(want - 1) / 2, d_taps, P, d_out);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

// Batch workspace: mel frames | window starts | partial embeddings (as many windows as frames) | trim RMS frames.
struct SpkBatchLayout { size_t starts, partials, rms, total; long long frames; };
static SpkBatchLayout spk_batch_layout(const mvb_spk_config* c, int max_batch, long long max_total_samples) {
  WsBump ws;
  SpkBatchLayout L;
  L.frames = max_batch + max_total_samples / c->hop;
  ws.take((size_t)L.frames * c->n_mels * 4);
  L.starts = ws.take((size_t)L.frames * 4);
  L.partials = ws.take((size_t)L.frames * 256 * 4);
  L.rms = ws.take((size_t)(max_batch + max_total_samples / TRIM_HOP) * 4);
  L.total = ws.end;
  return L;
}

static int spk_batch_capacity(int max_batch, long long max_total_samples) {
  if (max_batch < 1 || max_batch > SPK_MAX_BATCH)
    return mvb::set_error(MVB_ERR_ARG, "speaker batch: max_batch %d out of range [1, %d]", max_batch, SPK_MAX_BATCH);
  if (max_total_samples < 1 || max_total_samples > INT_MAX)
    return mvb::set_error(MVB_ERR_ARG, "speaker batch: max_total_samples %lld out of range [1, %d]", max_total_samples, INT_MAX);
  return MVB_OK;
}

extern "C" size_t mvb_spk_batch_workspace_bytes(const mvb_spk_config* c, int32_t max_batch, int64_t max_total_samples) {
  if (spk_validate(c) || spk_batch_capacity(max_batch, max_total_samples)) return 0;
  return spk_batch_layout(c, max_batch, max_total_samples).total;
}

extern "C" int mvb_spk_trim_batch(mvb_spk* h, int32_t n, const float* d_wav, const int32_t* n_samples, float top_db, void* d_batch_ws,
                                  int32_t max_batch, int64_t max_total_samples, int32_t* d_spans, void* stream) {
  if (!h || !d_wav || !n_samples || !d_batch_ws || !d_spans) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (int e = spk_batch_capacity(max_batch, max_total_samples)) return e;
  if (n < 1 || n > max_batch) return mvb::set_error(MVB_ERR_ARG, "trim: %d signals, capacity %d", n, max_batch);
  if (!(top_db > 0.f) || top_db > 3.0e38f) return mvb::set_error(MVB_ERR_ARG, "trim: top_db %g", (double)top_db);
  TrimSegs segs{};
  long long total = 0;
  int frames = 0, f_max = 0;
  for (int i = 0; i < n; ++i) {
    if (n_samples[i] < 1) return mvb::set_error(MVB_ERR_ARG, "trim: signal %d: %d samples", i, n_samples[i]);
    const int F = 1 + n_samples[i] / TRIM_HOP;
    segs.s[i] = TrimSeg{total, n_samples[i], frames};
    total += n_samples[i];
    frames += F;
    if (F > f_max) f_max = F;
  }
  if (total > max_total_samples) return mvb::set_error(MVB_ERR_ARG, "trim: %lld samples in all, capacity %lld", total, (long long)max_total_samples);
  const SpkBatchLayout L = spk_batch_layout(&h->cfg, max_batch, max_total_samples);
  float* rms = reinterpret_cast<float*>(reinterpret_cast<char*>(d_batch_ws) + L.rms);
  cudaStream_t s = (cudaStream_t)stream;
  k_trim_rms<<<dim3((f_max + 7) / 8, 1, n), 256, 0, s>>>(d_wav, segs, rms);
  MVB_CK(cudaGetLastError());
  k_trim_span<<<n, 256, 0, s>>>(rms, segs, (float)std::pow(10.0, -(double)top_db / 20.0), d_spans);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

extern "C" int mvb_spk_embed_batch(mvb_spk* h, int32_t n, const float* d_wav, const int64_t* wav_off, const int32_t* n_wav,
                                   const int32_t* starts, const int32_t* n_partials, void* d_batch_ws, int32_t max_batch,
                                   int64_t max_total_samples, float* d_embed, float* d_partials_out, void* stream) {
  if (!h || !d_wav || !wav_off || !n_wav || !starts || !n_partials || !d_batch_ws || !d_embed)
    return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (int e = spk_batch_capacity(max_batch, max_total_samples)) return e;
  if (n < 1 || n > max_batch) return mvb::set_error(MVB_ERR_ARG, "embed: %d utterances, capacity %d", n, max_batch);
  const mvb_spk_config& c = h->cfg;
  const SpkBatchLayout L = spk_batch_layout(&c, max_batch, max_total_samples);
  SpkSegs segs{};
  long long samples = 0, windows = 0;
  int frames = 0, f_max = 0;
  for (int i = 0; i < n; ++i) {
    if (wav_off[i] < 0 || n_wav[i] < 0 || n_partials[i] < 1)
      return mvb::set_error(MVB_ERR_ARG, "embed: utterance %d: offset %lld, %d samples, %d windows", i, (long long)wav_off[i],
                            n_wav[i], n_partials[i]);
    windows += n_partials[i];
    if (windows > L.frames) return mvb::set_error(MVB_ERR_ARG, "embed: more than %lld windows in all", L.frames);
    long long last = 0;
    for (long long w = windows - n_partials[i]; w < windows; ++w) {
      if (starts[w] < 0) return mvb::set_error(MVB_ERR_ARG, "embed: utterance %d: window start %d", i, starts[w]);
      if (starts[w] > last) last = starts[w];
    }
    // embed_utterance pads the waveform to the end of its last window: then every window lies in the spectrogram
    const long long padded = std::max((long long)n_wav[i], (last + c.partial_frames) * c.hop);
    if (padded > c.max_samples)
      return mvb::set_error(MVB_ERR_ARG, "embed: utterance %d: %lld samples with padding, capacity %d", i, padded, c.max_samples);
    const int F = 1 + (int)(padded / c.hop);
    segs.s[i] = SpkSeg{wav_off[i], n_wav[i], F, frames, (int)(windows - n_partials[i]), n_partials[i]};
    samples += padded;
    frames += F;
    if (F > f_max) f_max = F;
  }
  if (samples > max_total_samples)
    return mvb::set_error(MVB_ERR_ARG, "embed: %lld samples with padding in all, capacity %lld", samples, (long long)max_total_samples);
  std::vector<int> abs_starts(windows);                  // window starts offset into the utterance's mel block
  for (int i = 0; i < n; ++i)
    for (int w = 0; w < segs.s[i].n_part; ++w) abs_starts[segs.s[i].part_off + w] = segs.s[i].mel_off + starts[segs.s[i].part_off + w];
  char* ws = reinterpret_cast<char*>(d_batch_ws);
  float* mel = reinterpret_cast<float*>(ws);
  int* d_starts = reinterpret_cast<int*>(ws + L.starts);
  float* partials = reinterpret_cast<float*>(ws + L.partials);
  cudaStream_t s = (cudaStream_t)stream;
  MVB_CK(cudaMemcpyAsync(d_starts, abs_starts.data(), sizeof(int) * windows, cudaMemcpyHostToDevice, s));
  if (int e = spk_mel_segments(h, d_wav, segs, n, f_max, mel, s)) return e;
  if (int e = spk_lstm(h, mel, d_starts, frames, (int)windows, partials, nullptr, s)) return e;
  if (int e = spk_mean(partials, segs, n, d_embed, s)) return e;
  if (d_partials_out)
    MVB_CK(cudaMemcpyAsync(d_partials_out, partials, sizeof(float) * (size_t)windows * 256, cudaMemcpyDeviceToDevice, s));
  return MVB_OK;
}
