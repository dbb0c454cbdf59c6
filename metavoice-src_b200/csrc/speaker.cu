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

#include <vector>

#include "common.cuh"
#include "host.cuh"

using namespace mvb;

namespace {

constexpr int SPK_THREADS = 256;

// One frame per CTA: frame f covers samples [f*hop - n_fft/2, f*hop + n_fft/2) (center=True, zero padding).
__global__ void __launch_bounds__(SPK_THREADS) k_spk_mel(const float* __restrict__ wav, int n_samples, int n_fft, int hop,
                                                         const float* __restrict__ window, const float* __restrict__ cosT,
                                                         const float* __restrict__ sinT, const float* __restrict__ melfb,
                                                         int n_mels, float* __restrict__ mel) {
  extern __shared__ float sm[];
  float* frame = sm;                 // [n_fft]
  float* power = sm + n_fft;         // [n_fft/2 + 1]
  const int f = blockIdx.x, tid = threadIdx.x;
  const int n_bins = n_fft / 2 + 1;
  for (int n = tid; n < n_fft; n += SPK_THREADS) {
    const long long s = (long long)f * hop - n_fft / 2 + n;
    frame[n] = (s >= 0 && s < n_samples) ? wav[s] * window[n] : 0.f;
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
  for (int m = tid; m < n_mels; m += SPK_THREADS) {
    const float* fb = melfb + (size_t)m * n_bins;
    float acc = 0.f;
    for (int k = 0; k < n_bins; ++k) acc = fmaf(fb[k], power[k], acc);
    mel[(size_t)f * n_mels + m] = acc;
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

// raw = mean over the partial embeddings; embed = raw / ||raw||_2     (model.py:96-100)
__global__ void __launch_bounds__(SPK_THREADS) k_spk_mean(const float* __restrict__ partials, int P, float* __restrict__ out) {
  __shared__ float red[8];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float m = 0.f;
  for (int p = 0; p < P; ++p) m += partials[(size_t)p * 256 + tid];
  m /= (float)P;
  float ss = warp_sum(m * m);
  if (lane == 0) red[warp] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < 8; ++i) tot += red[i];
  out[tid] = m / sqrtf(tot);
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

static int spk_mel(mvb_spk* h, const float* d_wav, int n_samples, float* d_mel, cudaStream_t s) {
  const mvb_spk_config& c = h->cfg;
  const int n_frames = 1 + n_samples / c.hop;
  const size_t smem = (size_t)(c.n_fft + c.n_fft / 2 + 1) * 4;
  // tensors: 3 x {w_ih, w_hh, b}, linear w, linear b, mel filterbank, window, cos table, sin table
  k_spk_mel<<<n_frames, SPK_THREADS, smem, s>>>(d_wav, n_samples, c.n_fft, c.hop, h->w(12), h->w(13), h->w(14), h->w(11), c.n_mels, d_mel);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
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

static int spk_windows(mvb_spk* h, const float* d_mel, int n_frames, const int32_t* starts, int n_partials, float* d_partials,
                       float* d_trace, float* d_embed, cudaStream_t s) {
  if (int e = spk_check_windows(h, n_frames, starts, n_partials)) return e;
  const mvb_spk_config& c = h->cfg;
  if (starts) {
    MVB_CK(cudaMemcpyAsync(h->starts(), starts, sizeof(int) * n_partials, cudaMemcpyHostToDevice, s));
    SpkW W;
    for (int l = 0; l < 3; ++l) { W.w_ih[l] = h->w(3 * l); W.w_hh[l] = h->w(3 * l + 1); W.b[l] = h->w(3 * l + 2); }
    W.lw = h->w(9); W.lb = h->w(10);
    k_spk_lstm<<<n_partials, SPK_THREADS, 0, s>>>(d_mel, h->starts(), n_frames, c.partial_frames, c.n_mels, W, d_partials, d_trace);
    MVB_CK(cudaGetLastError());
  }
  if (d_embed) {
    k_spk_mean<<<1, SPK_THREADS, 0, s>>>(d_partials, n_partials, d_embed);
    MVB_CK(cudaGetLastError());
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
