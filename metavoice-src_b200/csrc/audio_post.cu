// On-device audio post-processing (SURVEY.md row N2): what `_save_audio` does on the host in the reference
// (fam/llm/decoders.py:40-47 -> audiocraft audio_write(strategy="loudness", loudness_compressor=True)):
//   integrated loudness (ITU-R BS.1770-4 as implemented by torchaudio.functional.loudness, the function audiocraft
//   calls: K-weighting = treble shelf + 38 Hz high-pass biquads, 400 ms blocks with 75 % overlap, absolute -70 LKFS and
//   relative -10 LU gates) -> gain to -14 LUFS -> tanh compressor -> clip -> PCM16.
// The waveform never leaves the device as fp32; the caller gets 16-bit samples (and the measured loudness).
//
// The two K-weighting biquads are recursive; they are evaluated in independent chunks, each warmed up over the
// preceding 4096 samples from a zero state (the slowest section, the 38 Hz high-pass, is a near-double pole whose impulse
// response there is 1.0e-14 at 24 kHz and 6e-6 at 48 kHz; tests/test_audio_post_ops_gpu.py), so the filter runs in
// ~6 K sequential steps instead of T.
//
// One launch set serves any number of signals: mvb_audio_post is a group of one, mvb_audio_post_batch launches its
// signals in groups of 32.
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "host.cuh"

using namespace mvb;

namespace {

struct Biquad { float b0, b1, b2, a1, a2; };   // normalised by a0

constexpr int KW_CHUNK = 2048, KW_WARM = 4096;

// Every kernel processes a group of n <= 32 signals concatenated in one buffer, passed by value as a segment list;
// blockIdx.y (k_loudness_gain: blockIdx.x) is the signal.  Signal i: samples [off, off + n) of the wav / PCM / K-weighted
// buffers, its n_blocks block energies, the whole-signal sum of squares and the 3 result scalars at e_off of the energy
// area.  Nothing a kernel computes for one signal depends on another.
constexpr int POST_GROUP = 32;
struct PostSeg { int n, off, n_blocks, e_off; };
struct PostSegs { PostSeg s[POST_GROUP]; };   // a kernel parameter (512 B): indexing it needs no device table

// y = clamp(hp(clamp(shelf(x))))   (torchaudio lfilter clamps each biquad's OUTPUT to [-1, 1], not its state);
// one thread per chunk of KW_CHUNK samples
__global__ void __launch_bounds__(128) k_kweight(const float* __restrict__ x, PostSegs segs, Biquad s, Biquad h, float* __restrict__ y) {
  const PostSeg g = segs.s[blockIdx.y];
  const int T = g.n, t0 = (blockIdx.x * blockDim.x + threadIdx.x) * KW_CHUNK;
  if (t0 >= T) return;
  x += g.off;
  y += g.off;
  const int start = max(0, t0 - KW_WARM), end = min(T, t0 + KW_CHUNK);
  float x1 = 0.f, x2 = 0.f, u1 = 0.f, u2 = 0.f;      // shelf: input / output history
  float c1 = 0.f, c2 = 0.f, v1 = 0.f, v2 = 0.f;      // high-pass: (clamped) input / output history
  for (int t = start; t < end; ++t) {
    const float xv = x[t];
    const float u = s.b0 * xv + s.b1 * x1 + s.b2 * x2 - s.a1 * u1 - s.a2 * u2;
    x2 = x1; x1 = xv; u2 = u1; u1 = u;
    const float c = fminf(fmaxf(u, -1.f), 1.f);
    const float v = h.b0 * c + h.b1 * c1 + h.b2 * c2 - h.a1 * v1 - h.a2 * v2;
    c2 = c1; c1 = c; v2 = v1; v1 = v;
    if (t >= t0) y[t] = fminf(fmaxf(v, -1.f), 1.f);
  }
}

// block b: mean of y^2 over [b*step, b*step + gate); block n_blocks: sum of x^2 over the whole signal (energy floor test)
__global__ void __launch_bounds__(256) k_block_energy(const float* __restrict__ y, const float* __restrict__ x, PostSegs segs, int gate,
                                                      int step, float* __restrict__ energy) {
  __shared__ float red[8];
  const PostSeg g = segs.s[blockIdx.y];
  const int b = blockIdx.x;
  if (b > g.n_blocks) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* src = b < g.n_blocks ? y + g.off + (size_t)b * step : x + g.off;
  const int n = b < g.n_blocks ? gate : g.n;
  float acc = 0.f;
  for (int i = tid; i < n; i += 256) acc = fmaf(src[i], src[i], acc);
  acc = warp_sum(acc);
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    energy[g.e_off + b] = b < g.n_blocks ? t / (float)gate : t;
  }
}

// gating + gain (one thread: <= 16000 blocks).  out[0] = LKFS, out[1] = linear gain, out[2] = 1 when the compressor may
// run.  Below the energy floor: LKFS = -inf, gain 1, no compressor (audiocraft's normalize_loudness leaves the signal
// untouched).  Where the meter is undefined -- non-finite input, no complete block, or every block gated (torchaudio
// returns NaN or raises there, and normalize_loudness fails its finiteness assert) -- LKFS = NaN, gain 1, no compressor,
// so that no NaN reaches the PCM.
__device__ __forceinline__ void loudness_gain(const float* __restrict__ energy, int n_blocks, int T, float headroom_db, float energy_floor,
                                              float* __restrict__ out) {
  out[1] = 1.f; out[2] = 0.f;
  const float rms = sqrtf(energy[n_blocks] / (float)T);
  if (!isfinite(rms)) { out[0] = NAN; return; }
  if (rms < energy_floor) { out[0] = -INFINITY; return; }
  const float bias = -0.691f, gamma_abs = -70.f;
  float sum = 0.f; int cnt = 0;
  for (int b = 0; b < n_blocks; ++b) {
    const float l = bias + 10.f * log10f(energy[b]);
    if (l > gamma_abs) { sum += energy[b]; ++cnt; }
  }
  if (cnt == 0) { out[0] = NAN; return; }
  const float gamma_rel = bias + 10.f * log10f(sum / (float)cnt) - 10.f;
  sum = 0.f; cnt = 0;
  for (int b = 0; b < n_blocks; ++b) {
    const float l = bias + 10.f * log10f(energy[b]);
    if (l > gamma_abs && l > gamma_rel) { sum += energy[b]; ++cnt; }
  }
  if (cnt == 0) { out[0] = NAN; return; }
  const float lkfs = bias + 10.f * log10f(sum / (float)cnt);
  out[0] = lkfs;
  out[1] = powf(10.f, (-headroom_db - lkfs) / 20.f);
  out[2] = 1.f;
}

// one CTA per signal: its result scalars, and {LKFS, gain} of signal blockIdx.x to lkfs_gain when given
__global__ void k_loudness_gain(float* __restrict__ energy, PostSegs segs, float headroom_db, float energy_floor,
                                float* __restrict__ lkfs_gain) {
  if (threadIdx.x != 0) return;
  const PostSeg g = segs.s[blockIdx.x];
  float* res = energy + g.e_off + g.n_blocks + 1;
  loudness_gain(energy + g.e_off, g.n_blocks, g.n, headroom_db, energy_floor, res);
  if (lkfs_gain) { lkfs_gain[2 * blockIdx.x] = res[0]; lkfs_gain[2 * blockIdx.x + 1] = res[1]; }
}

// out = clip(tanh(gain * x)) -> PCM16 (round to nearest even, like numpy's round in audio_out.py / torchaudio.save).
// A NaN sample is written as 0 (fmaxf would otherwise turn it into -1).  Grid-stride over the signal's samples.
__global__ void __launch_bounds__(256) k_apply_pcm16(const float* __restrict__ x, PostSegs segs, const float* __restrict__ energy,
                                                     int compressor, short* __restrict__ pcm, float* __restrict__ wav_out) {
  const PostSeg g = segs.s[blockIdx.y];
  const float* res = energy + g.e_off + g.n_blocks + 1;
  const float gain = res[1];
  const bool comp = compressor && res[2] != 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += gridDim.x * blockDim.x) {
    float v = gain * x[g.off + i];
    if (comp) v = tanhf(v);
    v = isnan(v) ? 0.f : fminf(fmaxf(v, -1.f), 1.f);
    if (wav_out) wav_out[g.off + i] = v;
    pcm[g.off + i] = (short)__float2int_rn(v * 32767.f);
  }
}

static Biquad treble_shelf(double sr, double gain_db, double f0, double Q) {   // torchaudio.functional.treble_biquad
  const double w0 = 2 * M_PI * f0 / sr, alpha = sin(w0) / 2 / Q, A = exp(gain_db / 40 * log(10.0));
  const double t1 = 2 * sqrt(A) * alpha, t2 = (A - 1) * cos(w0), t3 = (A + 1) * cos(w0);
  const double b0 = A * ((A + 1) + t2 + t1), b1 = -2 * A * ((A - 1) + t3), b2 = A * ((A + 1) + t2 - t1);
  const double a0 = (A + 1) - t2 + t1, a1 = 2 * ((A - 1) - t3), a2 = (A + 1) - t2 - t1;
  return Biquad{(float)(b0 / a0), (float)(b1 / a0), (float)(b2 / a0), (float)(a1 / a0), (float)(a2 / a0)};
}
static Biquad highpass(double sr, double f0, double Q) {                      // torchaudio.functional.highpass_biquad
  const double w0 = 2 * M_PI * f0 / sr, alpha = sin(w0) / 2 / Q;
  const double b0 = (1 + cos(w0)) / 2, b1 = -1 - cos(w0), b2 = b0, a0 = 1 + alpha, a1 = -2 * cos(w0), a2 = 1 - alpha;
  return Biquad{(float)(b0 / a0), (float)(b1 / a0), (float)(b2 / a0), (float)(a1 / a0), (float)(a2 / a0)};
}

// Workspace for n samples: K-weighted copy | ENERGY_BYTES of block energies + result scalars (at energy_offset(n))
constexpr size_t ENERGY_BYTES = 65536;
size_t energy_offset(size_t n) { WsBump ws; ws.take(n * 4); return ws.take(ENERGY_BYTES); }

// Gating blocks of 400 ms with 75 % overlap: the number of complete blocks, their length and hop in samples
int gate_blocks(int n_samples, int sample_rate, int* gate, int* step) {
  *gate = (int)lround(0.4 * sample_rate);
  *step = (int)lround(*gate * 0.25);
  return n_samples >= *gate ? (n_samples - *gate) / *step + 1 : 0;
}

// The launch sequence over one group of n <= POST_GROUP validated signals: y = the K-weighted copy and energy = the
// energy area the segments' offsets index; d_lkfs_gain (optional) receives the group's {LKFS, gain} pairs.
int post_group(const float* d_wav, const PostSegs& g, int n, int sample_rate, float loudness_headroom_db, int loudness_compressor,
               float* y, float* energy, int16_t* d_pcm16, float* d_wav_out, float* d_lkfs_gain, cudaStream_t s) {
  int gate, step, max_n = 0, max_blocks = 0;
  gate_blocks(1, sample_rate, &gate, &step);
  for (int i = 0; i < n; ++i) {
    max_n = max(max_n, g.s[i].n);
    max_blocks = max(max_blocks, g.s[i].n_blocks);
  }
  const int chunks = (max_n + KW_CHUNK - 1) / KW_CHUNK;
  k_kweight<<<dim3((chunks + 127) / 128, n), 128, 0, s>>>(d_wav, g, treble_shelf(sample_rate, 4.0, 1500.0, 1.0 / sqrt(2.0)),
                                                        highpass(sample_rate, 38.0, 0.5), y);
  MVB_CK(cudaGetLastError());
  k_block_energy<<<dim3(max_blocks + 1, n), 256, 0, s>>>(y, d_wav, g, gate, step, energy);
  MVB_CK(cudaGetLastError());
  k_loudness_gain<<<n, 32, 0, s>>>(energy, g, loudness_headroom_db, 2e-3f, d_lkfs_gain);
  MVB_CK(cudaGetLastError());
  const int per_signal = max(1, min(GRID_STRIDE_CTAS * 4, (max_n + 2047) / 2048));
  k_apply_pcm16<<<dim3(per_signal, n), 256, 0, s>>>(d_wav, g, energy, loudness_compressor, d_pcm16, d_wav_out);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

}  // namespace

extern "C" size_t mvb_audio_post_workspace_bytes(int32_t max_samples) {
  if (max_samples < 1) return 0;
  return energy_offset(max_samples) + ENERGY_BYTES;
}

// A group of one signal: y at 0, its energies and results at energy_offset(n_samples) (one signal needs at most
// 16,000 floats there, which ENERGY_BYTES holds).
extern "C" int mvb_audio_post(const float* d_wav, int32_t n_samples, int32_t sample_rate, float loudness_headroom_db,
                              int32_t loudness_compressor, void* d_workspace, int16_t* d_pcm16, float* d_wav_out,
                              float* d_lkfs_gain, void* stream) {
  if (!d_wav || !d_workspace || !d_pcm16) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (n_samples < 1 || sample_rate < 8000) return mvb::set_error(MVB_ERR_ARG, "audio_post: bad length / sample rate");
  int gate, step;
  const int n_blocks = gate_blocks(n_samples, sample_rate, &gate, &step);
  if (n_blocks + 4 > 16000) return mvb::set_error(MVB_ERR_UNSUPPORTED, "audio_post: signal too long for the workspace");
  PostSegs g{};
  g.s[0] = PostSeg{n_samples, 0, n_blocks, 0};
  char* ws = reinterpret_cast<char*>(d_workspace);
  return post_group(d_wav, g, 1, sample_rate, loudness_headroom_db, loudness_compressor, reinterpret_cast<float*>(ws),
                    reinterpret_cast<float*>(ws + energy_offset(n_samples)), d_pcm16, d_wav_out, d_lkfs_gain, (cudaStream_t)stream);
}

// ---- batched post ----------------------------------------------------------------------------------------------------
// Workspace: K-weighted copy [max_total_samples] | energy area.  At >= 8 kHz a gating hop is >= 800 samples, so signal i
// needs at most n_i / 800 + 1 block energies + 1 sum + 3 results.
constexpr int POST_MAX_BATCH = 65535;   // the capacity range of the ABI (signals are launched in groups of POST_GROUP)

struct PostBatchLayout { size_t energy, total; };

static PostBatchLayout post_batch_layout(int max_batch, int max_total_samples) {
  PostBatchLayout L;
  WsBump ws;
  ws.take((size_t)max_total_samples * 4);
  L.energy = ws.take(((size_t)max_total_samples / 800 + 5 * (size_t)max_batch) * 4);
  L.total = ws.end;
  return L;
}

extern "C" size_t mvb_audio_post_batch_workspace_bytes(int32_t max_batch, int32_t max_total_samples) {
  if (max_batch < 1 || max_batch > POST_MAX_BATCH || max_total_samples < 1) return 0;
  return post_batch_layout(max_batch, max_total_samples).total;
}

// mvb_audio_post over n concatenated signals, one launch set per group of POST_GROUP signals; signal i's outputs equal
// mvb_audio_post's on it alone.
extern "C" int mvb_audio_post_batch(const float* d_wav, int32_t n, const int32_t* n_samples, int32_t sample_rate,
                                    float loudness_headroom_db, int32_t loudness_compressor, void* d_workspace, int32_t max_batch,
                                    int32_t max_total_samples, int16_t* d_pcm16, float* d_wav_out, float* d_lkfs_gain, void* stream) {
  if (!d_wav || !n_samples || !d_workspace || !d_pcm16) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (max_batch < 1 || max_batch > POST_MAX_BATCH || max_total_samples < 1)
    return mvb::set_error(MVB_ERR_ARG, "audio_post batch: bad capacity (%d signals, %d samples)", max_batch, max_total_samples);
  if (n < 1 || n > max_batch) return mvb::set_error(MVB_ERR_ARG, "audio_post batch: %d signals, capacity %d", n, max_batch);
  if (sample_rate < 8000) return mvb::set_error(MVB_ERR_ARG, "audio_post: bad length / sample rate");
  std::vector<PostSeg> segs(n);
  long long total = 0, e_total = 0;
  for (int i = 0; i < n; ++i) {
    if (n_samples[i] < 1) return mvb::set_error(MVB_ERR_ARG, "audio_post batch: signal %d: bad length %d", i, n_samples[i]);
    int gate, step;
    const int nb = gate_blocks(n_samples[i], sample_rate, &gate, &step);
    if (nb + 4 > 16000) return mvb::set_error(MVB_ERR_UNSUPPORTED, "audio_post: signal %d too long for the workspace", i);
    segs[i] = PostSeg{n_samples[i], (int)total, nb, (int)e_total};
    total += n_samples[i];
    e_total += nb + 4;
  }
  if (total > max_total_samples)
    return mvb::set_error(MVB_ERR_ARG, "audio_post batch: %lld samples in all, capacity %d", total, max_total_samples);
  char* ws = reinterpret_cast<char*>(d_workspace);
  float* energy = reinterpret_cast<float*>(ws + post_batch_layout(max_batch, max_total_samples).energy);
  for (int g0 = 0; g0 < n; g0 += POST_GROUP) {
    const int k = min(POST_GROUP, n - g0);
    PostSegs g{};
    std::copy(segs.begin() + g0, segs.begin() + g0 + k, g.s);
    if (int e = post_group(d_wav, g, k, sample_rate, loudness_headroom_db, loudness_compressor, reinterpret_cast<float*>(ws), energy,
                           d_pcm16, d_wav_out, d_lkfs_gain ? d_lkfs_gain + 2 * g0 : nullptr, (cudaStream_t)stream))
      return e;
  }
  return MVB_OK;
}

extern "C" int mvb_audio_post_test(const float* d_wav, int32_t n_samples, int32_t sample_rate, float loudness_headroom_db,
                                   int32_t loudness_compressor, int16_t* d_pcm16, float* d_wav_out, float* d_y, float* d_energy,
                                   float* d_res, int32_t* n_blocks_out, void* stream) {
  if (!d_y || !d_energy || !d_res || !n_blocks_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (n_samples < 1 || sample_rate < 8000) return mvb::set_error(MVB_ERR_ARG, "audio_post: bad length / sample rate");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t bytes = mvb_audio_post_workspace_bytes(n_samples);
  char* ws = nullptr;
  MVB_CK(cudaMalloc(&ws, bytes));
  int rc = mvb_audio_post(d_wav, n_samples, sample_rate, loudness_headroom_db, loudness_compressor, ws, d_pcm16, d_wav_out,
                          nullptr, stream);
  if (rc == MVB_OK) {
    int gate, step;
    const int n_blocks = gate_blocks(n_samples, sample_rate, &gate, &step);
    const float* energy = reinterpret_cast<const float*>(ws + energy_offset(n_samples));
    cudaError_t e = cudaMemcpyAsync(d_y, ws, (size_t)n_samples * 4, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_energy, energy, (size_t)(n_blocks + 1) * 4, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_res, energy + n_blocks + 1, 3 * 4, cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) rc = mvb::set_error(MVB_ERR_CUDA, "mvb_audio_post_test: %s", cudaGetErrorString(e));
    *n_blocks_out = n_blocks;
  }
  const cudaError_t e = cudaStreamSynchronize(s);   // (also on an error path: the buffer is freed only once unused)
  if (rc == MVB_OK && e != cudaSuccess) rc = mvb::set_error(MVB_ERR_CUDA, "mvb_audio_post_test: %s", cudaGetErrorString(e));
  cudaFree(ws);
  return rc;
}
