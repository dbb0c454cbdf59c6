// Multi-band-diffusion vocoder (SURVEY.md row a17, second half): what `mbd.tokens_to_wav` (fam/llm/decoders.py:84-85 ->
// audiocraft 1.2.0 MultiBandDiffusion) evaluates after the EnCodec decode of csrc/vocoder.cu:
//     wav = sum over the band models of  DiffusionProcess.generate(condition = codec latent, 20 sampler steps each)
//     out = re_eq(wav, ref = EnCodec waveform, 32 mel bands)
// PARITY UNPINNED: audiocraft / julius / mbd_comp_8.pt are not in the image; the algorithm is restated from the paper
// (arXiv 2308.02560) and the audiocraft modules named in oracle/mbd_port.py against a PARAMETRISED configuration
// (mvb_mbd_config); the GPU code is tested against that restatement.
//
// Activations are [C][T] fp32 (time contiguous), fp32 arithmetic throughout (the reference forces fp32 autocast for the
// vocoder, decoders.py:84).  Every convolution streams its input window through a shared-memory line buffer with the
// preceding GroupNorm + ReLU applied on the fly (statistics from a reduction kernel), keeps an 8-channel x {1,2,4}-sample
// register tile per thread and fuses bias / residual / step-embedding adds into the epilogue.  The band splitters
// (julius.SplitBands: windowed-sinc low-pass banks, 629 / 2893 taps) are direct FIR kernels.
#include <cuda_runtime.h>
#include <math.h>

#include <vector>

#include "common.cuh"
#include "host.cuh"
#include "mbd_tc.cuh"
#include "tc_gemm_host.cuh"

using namespace mvb;

namespace {

// ---- GroupNorm statistics: stats[2g] = mean, stats[2g+1] = 1/sqrt(var + eps) over (C/groups) x T  (nn.GroupNorm, biased variance).
// Two stages so that a 4-group norm still fills the machine: GN_SPLIT CTAs per group write fp64 partial sums, one small CTA
// adds them in a fixed order (run-to-run deterministic).
constexpr int GN_SPLIT = 64;
constexpr float GN_EPS = 1e-5f;   // nn.GroupNorm's default
__global__ void __launch_bounds__(256) k_gn_partial(const float* __restrict__ x, size_t n, double* __restrict__ part) {
  __shared__ double rs[8], rq[8];
  const int g = blockIdx.x, sp = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* p = x + (size_t)g * n;
  const size_t lo = n * sp / GN_SPLIT, hi = n * (sp + 1) / GN_SPLIT;
  double s = 0.0, q = 0.0;
  for (size_t i = lo + tid; i < hi; i += 256) {
    const double v = p[i];
    s += v;
    q += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (lane == 0) { rs[warp] = s; rq[warp] = q; }
  __syncthreads();
  if (tid == 0) {
    double S = 0.0, Q = 0.0;
    for (int i = 0; i < 8; ++i) { S += rs[i]; Q += rq[i]; }
    part[2 * (g * GN_SPLIT + sp)] = S;
    part[2 * (g * GN_SPLIT + sp) + 1] = Q;
  }
}
// one warp per group: lane i adds partials i and i + 32, then a fixed-shape butterfly (deterministic)
__global__ void k_gn_final(const double* __restrict__ part, int groups, double n, float eps, float* __restrict__ stats) {
  const int g = blockIdx.x, lane = threadIdx.x;
  double S = 0.0, Q = 0.0;
  for (int i = lane; i < GN_SPLIT; i += 32) { S += part[2 * (g * GN_SPLIT + i)]; Q += part[2 * (g * GN_SPLIT + i) + 1]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    S += __shfl_xor_sync(0xffffffffu, S, o);
    Q += __shfl_xor_sync(0xffffffffu, Q, o);
  }
  if (lane == 0) {
    const double mean = S / n, var = Q / n - mean * mean;
    stats[2 * g] = (float)mean;
    stats[2 * g + 1] = (float)(1.0 / sqrt((var > 0.0 ? var : 0.0) + (double)eps));
  }
}

struct ConvP {
  const float* x; int Cin, Tin;
  const float* w; const float* bias;          // w [Cout][Cin][K]; bias may be null
  float* y; int Cout, Tout;
  int dil, pad;
  const float* gn_stats; const float* gn_w; const float* gn_b; int groups;   // input transform relu(GN(x)) when gn_stats != null
  const float* resid;                           // optional [Cout][Tout] added to the output
  const float* emb;                             // optional [Cout] added to the output (step embedding)
};

// Conv1d with zero padding, stride STRIDE, dilation p.dil.  Tile: 32 output channels x (64 * TPT) outputs, 16 input channels per pass.
template <int K, int STRIDE, int TPT>
__global__ void __launch_bounds__(256) k_mbd_conv(const ConvP p) {
  constexpr int CI = 16, CO = 32, TT = 64 * TPT, LBMAX = 296;
  __shared__ float xs[CI][LBMAX];
  __shared__ float ws[CO][CI][K];
  const int t0 = blockIdx.x * TT, co0 = blockIdx.y * CO;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int LB = (TT - 1) * STRIDE + (K - 1) * p.dil + 1;
  const int in0 = t0 * STRIDE - p.pad;
  const int cpg = p.gn_stats ? p.Cin / p.groups : 1;
  float acc[8][TPT];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TPT; ++j) acc[i][j] = 0.f;
  for (int c0 = 0; c0 < p.Cin; c0 += CI) {
    __syncthreads();
    for (int i = threadIdx.x; i < CI * LB; i += 256) {
      const int ci = i / LB, tt = i - ci * LB;
      const int c = c0 + ci, t = in0 + tt;
      float v = 0.f;
      if (c < p.Cin && t >= 0 && t < p.Tin) {
        v = p.x[(size_t)c * p.Tin + t];
        if (p.gn_stats) {
          const int g = c / cpg;
          v = fmaxf((v - p.gn_stats[2 * g]) * p.gn_stats[2 * g + 1] * p.gn_w[c] + p.gn_b[c], 0.f);
        }
      }
      xs[ci][tt] = v;
    }
    for (int i = threadIdx.x; i < CO * CI * K; i += 256) {
      const int co = i / (CI * K), r = i - co * (CI * K), ci = r / K, k = r - ci * K;
      ws[co][ci][k] = (co0 + co < p.Cout && c0 + ci < p.Cin) ? p.w[((size_t)(co0 + co) * p.Cin + c0 + ci) * K + k] : 0.f;
    }
    __syncthreads();
#pragma unroll 2
    for (int ci = 0; ci < CI; ++ci) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        float xv[TPT];
#pragma unroll
        for (int j = 0; j < TPT; ++j) xv[j] = xs[ci][(tx * TPT + j) * STRIDE + k * p.dil];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float wv = ws[ty * 8 + i][ci][k];
#pragma unroll
          for (int j = 0; j < TPT; ++j) acc[i][j] = fmaf(wv, xv[j], acc[i][j]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int co = co0 + ty * 8 + i;
    if (co >= p.Cout) continue;
    const float add = (p.bias ? p.bias[co] : 0.f) + (p.emb ? p.emb[co] : 0.f);
#pragma unroll
    for (int j = 0; j < TPT; ++j) {
      const int t = t0 + tx * TPT + j;
      if (t < p.Tout) {
        float v = acc[i][j] + add;
        if (p.resid) v += p.resid[(size_t)co * p.Tout + t];
        p.y[(size_t)co * p.Tout + t] = v;
      }
    }
  }
}

// ConvTranspose1d(K = 2 * S, stride S, padding pad, no bias) of relu(GN(x)):  y[co][tau] = sum_ci sum_k w[ci][co][k] f(x[ci][t]),
// tau = t * S - pad + k.  Each output has exactly two taps (k0 = (tau + pad) mod S and k0 + S).  Tile: 32 co x 256 outputs.
template <int S>
__global__ void __launch_bounds__(256) k_mbd_convtr(const ConvP p) {
  constexpr int K = 2 * S, CI = 16, CO = 32, TT = 256, TI = TT / S + 2;
  __shared__ float xs[CI][TI];
  __shared__ float ws[CI][CO][K];
  const int o0 = blockIdx.x * TT, co0 = blockIdx.y * CO;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int tin0 = (o0 + p.pad) / S - 1;             // first input sample any output of this tile may touch
  const int cpg = p.gn_stats ? p.Cin / p.groups : 1;
  int tl[4], kk[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int o = o0 + tx + 64 * j + p.pad;
    kk[j] = o % S;                                    // first tap; the second is kk + S with input index - 1
    tl[j] = o / S - tin0;
  }
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int c0 = 0; c0 < p.Cin; c0 += CI) {
    __syncthreads();
    for (int i = threadIdx.x; i < CI * TI; i += 256) {
      const int ci = i / TI, tt = i - ci * TI;
      const int c = c0 + ci, t = tin0 + tt;
      float v = 0.f;
      if (c < p.Cin && t >= 0 && t < p.Tin) {
        v = p.x[(size_t)c * p.Tin + t];
        if (p.gn_stats) {
          const int g = c / cpg;
          v = fmaxf((v - p.gn_stats[2 * g]) * p.gn_stats[2 * g + 1] * p.gn_w[c] + p.gn_b[c], 0.f);
        }
      }
      xs[ci][tt] = v;
    }
    for (int i = threadIdx.x; i < CI * CO * K; i += 256) {
      const int ci = i / (CO * K), r = i - ci * (CO * K), co = r / K, k = r - co * K;
      ws[ci][co][k] = (c0 + ci < p.Cin && co0 + co < p.Cout) ? p.w[((size_t)(c0 + ci) * p.Cout + co0 + co) * K + k] : 0.f;
    }
    __syncthreads();
    for (int ci = 0; ci < CI; ++ci) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float e1 = xs[ci][tl[j]], e0 = xs[ci][tl[j] - 1];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float* wp = &ws[ci][ty * 8 + i][0];
          acc[i][j] = fmaf(wp[kk[j]], e1, fmaf(wp[kk[j] + S], e0, acc[i][j]));
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int co = co0 + ty * 8 + i;
    if (co >= p.Cout) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = o0 + tx + 64 * j;
      if (o < p.Tout) p.y[(size_t)co * p.Tout + o] = acc[i][j];
    }
  }
}

// out[c][t] = z[c][t] (cropped to Ts) + s[c][t]
__global__ void k_add_crop(const float* __restrict__ z, int Tz, const float* __restrict__ s, int Ts, int C, float* __restrict__ out) {
  const size_t n = (size_t)C * Ts;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / Ts), t = (int)(i - (size_t)c * Ts);
    out[i] = z[(size_t)c * Tz + t] + s[i];
  }
}
// z[c][t] += cond[c][nearest(t)]   (F.interpolate(cond, Tz), mode "nearest": src = floor(dst * Tf / Tz) in fp32)
__global__ void k_add_interp(float* __restrict__ z, int Tz, const float* __restrict__ cond, int Tf, int C) {
  const size_t n = (size_t)C * Tz;
  const float scale = (float)Tf / (float)Tz;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / Tz), t = (int)(i - (size_t)c * Tz);
    const int src = min((int)floorf((float)t * scale), Tf - 1);
    z[i] += cond[(size_t)c * Tf + src];
  }
}
// NoiseSchedule.generate_subsampled, one step: cur = clamp((cur - a * est * ns) * b + sigma * noise * ns)
__global__ void k_sched_step(float* __restrict__ cur, const float* __restrict__ est, const float* __restrict__ noise, float a, float b,
                             float sigma, float ns, float clip, int T) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < T; i += gridDim.x * blockDim.x) {
    float v = (cur[i] - a * (est[i] * ns)) * b;
    if (sigma > 0.f) v += sigma * noise[i] * ns;
    if (clip > 0.f) v = fminf(fmaxf(v, -clip), clip);
    cur[i] = v;
  }
}
// wav0[t] = sum_m wav_m[t] over the per-model blocks (block stride in floats), in model order
__global__ void k_sum_blocks(float* __restrict__ wav0, size_t blk_floats, int n, int T) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < T; i += gridDim.x * blockDim.x) {
    float a = wav0[i];
    for (int m = 1; m < n; ++m) a += wav0[(size_t)m * blk_floats + i];
    wav0[i] = a;
  }
}
__global__ void k_scale_copy(const float* __restrict__ src, float s, float* __restrict__ dst, int T) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < T; i += gridDim.x * blockDim.x) dst[i] = src[i] * s;
}
// standard normal draws (Box-Muller over Philox) when the caller supplies no noise
__global__ void k_randn(float* __restrict__ out, int T, unsigned long long seed, unsigned stream_id) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (T + 1) / 2; i += gridDim.x * blockDim.x) {
    const uint4 r = philox4x32_10(make_uint4((unsigned)i, stream_id, 0x6d6264u, 0u), make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
    const float u1 = ((float)(r.x >> 8) + 0.5f) * (1.0f / 16777216.0f), u2 = ((float)(r.y >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float rad = sqrtf(-2.f * logf(u1));
    float sn, cs;
    sincospif(2.f * u2, &sn, &cs);
    out[2 * i] = rad * cs;
    if (2 * i + 1 < T) out[2 * i + 1] = rad * sn;
  }
}

// julius.LowPassFilters with replicate padding: low[f][t] = sum_j bank[f][j] * x[clamp(t + j - half)].  One CTA = 1024 outputs of two
// filters: every thread keeps 4 outputs (t, t+256, t+512, t+768) x 2 filters in registers, so one tap costs 4 conflict-free x
// reads + 2 broadcast coefficient reads for 8 FMAs (the direct form was 2 shared-memory reads per FMA).
constexpr int FIR_TT = 1024;
// dynamic shared memory for L taps (the x window [FIR_TT + L - 1] and two filters [L]); the H100 opt-in maximum of 227 KB
// bounds L at 19029 taps, far above the 5921 of a 64-band bank at 24 kHz
constexpr size_t FIR_SMEM_MAX = 227 * 1024;
static size_t fir_smem_bytes(int L) { return (size_t)(FIR_TT + 3 * (size_t)L) * 4; }
__global__ void __launch_bounds__(256) k_fir_bank(const float* __restrict__ x, int T, const float* __restrict__ bank, int L, int nf,
                                                  float* __restrict__ low) {
  extern __shared__ float sm[];
  float* xs = sm;                       // [FIR_TT + L - 1]
  float* f0s = sm + FIR_TT + L - 1;     // [L]
  float* f1s = f0s + L;                 // [L]
  const int t0 = blockIdx.x * FIR_TT, f0 = blockIdx.y * 2, f1 = f0 + 1, half = (L - 1) / 2;
  const bool two = f1 < nf;
  for (int i = threadIdx.x; i < FIR_TT + L - 1; i += 256) {
    int t = t0 + i - half;
    t = t < 0 ? 0 : (t >= T ? T - 1 : t);
    xs[i] = x[t];
  }
  for (int i = threadIdx.x; i < L; i += 256) {
    f0s[i] = bank[(size_t)f0 * L + i];
    f1s[i] = two ? bank[(size_t)f1 * L + i] : 0.f;
  }
  __syncthreads();
  float a[4] = {0.f, 0.f, 0.f, 0.f}, b[4] = {0.f, 0.f, 0.f, 0.f};
  const float* xp = xs + threadIdx.x;
#pragma unroll 4
  for (int j = 0; j < L; ++j) {
    const float c0 = f0s[j], c1 = f1s[j];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float xv = xp[j + 256 * k];
      a[k] = fmaf(c0, xv, a[k]);
      b[k] = fmaf(c1, xv, b[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int t = t0 + threadIdx.x + 256 * k;
    if (t < T) {
      low[(size_t)f0 * T + t] = a[k];
      if (two) low[(size_t)f1 * T + t] = b[k];
    }
  }
}
// band b of SplitBands from the low-passed copies: b = 0: low[0]; 0 < b < n-1: low[b] - low[b-1]; b = n-1: x - low[n-2]
__device__ __forceinline__ float band_at(const float* low, const float* x, int T, int n_bands, int b, int t) {
  const float hi = b == n_bands - 1 ? x[t] : low[(size_t)b * T + t];
  const float lo = b == 0 ? 0.f : low[(size_t)(b - 1) * T + t];
  return hi - lo;
}
// per band: sum and sum of squares (double) -> unbiased std like Tensor.std()
__global__ void __launch_bounds__(256) k_band_std(const float* __restrict__ low, const float* __restrict__ x, int T, int n_bands, float* __restrict__ stdv) {
  __shared__ double rs[8], rq[8];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  double s = 0.0, q = 0.0;
  for (int t = tid; t < T; t += 256) {
    const double v = band_at(low, x, T, n_bands, b, t);
    s += v;
    q += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (lane == 0) { rs[warp] = s; rq[warp] = q; }
  __syncthreads();
  if (tid == 0) {
    double S = 0.0, Q = 0.0;
    for (int i = 0; i < 8; ++i) { S += rs[i]; Q += rq[i]; }
    const double var = (Q - S * S / (double)T) / (double)(T - 1);
    stdv[b] = (float)sqrt(var > 0.0 ? var : 0.0);
  }
}
// out[t] (+)= sum_b scale[b] * band_b[t] + shift[b];  scale = num[b] / den[b] when den != null (re_eq), else num[b]
__global__ void __launch_bounds__(256) k_band_mix(const float* __restrict__ low, const float* __restrict__ x, int T, int n_bands,
                                                  const float* __restrict__ num, const float* __restrict__ den,
                                                  const float* __restrict__ shift, float* __restrict__ out, int accumulate) {
  __shared__ float sc[64], sh[64];
  if ((int)threadIdx.x < n_bands) {
    sc[threadIdx.x] = den ? num[threadIdx.x] / den[threadIdx.x] : num[threadIdx.x];
    sh[threadIdx.x] = shift ? shift[threadIdx.x] : 0.f;
  }
  __syncthreads();
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < T; t += gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int b = 0; b < n_bands; ++b) acc += band_at(low, x, T, n_bands, b, t) * sc[b] + sh[b];
    out[t] = accumulate ? out[t] + acc : acc;
  }
}

__global__ void k_gn_relu_inplace(float* x, int C, int T, int cpg, const float* st, const float* gw, const float* gb) {
  const size_t n = (size_t)C * T;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / T), g = c / cpg;
    x[i] = fmaxf((x[i] - st[2 * g]) * st[2 * g + 1] * gw[c] + gb[c], 0.f);
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// Workspace layout, a function of the config alone (the MVB_MBD_CUDA_CORES / MVB_MBD_ONE_STREAM options included)
struct MbdWs {
  size_t cur, est, noise, wav, cond, gn, gn_part, stdv, low, skip[8], tmp[3], xt_hi, xt_lo;   // offsets inside one activation block
  size_t blk, wpack, total;   // block size; the packed taps follow n_blk blocks (one block per concurrently running band model)
  int n_blk;
  bool tc;                    // convolutions with input widths >= 32 run on the tensor cores
};

struct mvb_mbd {
  mvb_mbd_config cfg;
  const char* arena;
  std::vector<uint64_t> off;
  char* ws;
  std::vector<int> ch;       // channels per level
  int per_model = 0;         // tensors per band model
  // tensor-core path (mbd_tc.cuh): packed bf16 taps + their tensor maps, by weight tensor index
  struct TcW { CUtensorMap tmA; int Cin, Cout, K; };
  char* base = nullptr;      // activation block of the band model whose kernels are being enqueued (host-side cursor)
  cudaStream_t st[8] = {};   // one stream per band model (n_blk > 1)
  cudaEvent_t ev_fork = nullptr, ev_join[8] = {};
  MbdWs L{};
  std::vector<int> tc_of;    // [n tensors] -> index into tcw, or -1 (CUDA-core path)
  std::vector<TcW> tcw;
  const float* w(int i) const { return reinterpret_cast<const float*>(arena + off[i]); }
};

static int mbd_validate(const mvb_mbd_config* c) {
  if (!c) return mvb::set_error(MVB_ERR_ARG, "null config");
  if (c->depth < 1 || c->depth > 6 || c->res_blocks < 1 || c->res_blocks > 4 || c->n_models < 1 || c->n_models > 8)
    return mvb::set_error(MVB_ERR_ARG, "mbd: depth / res_blocks / n_models out of range");
  if (!((c->kernel == 8 && c->stride == 4) || (c->kernel == 4 && c->stride == 2)))
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "mbd: (kernel, stride) must be (8, 4) or (4, 2)");
  if (c->chin != 1) return mvb::set_error(MVB_ERR_UNSUPPORTED, "mbd: mono waveforms only (chin = 1)");
  // the workspace holds GroupNorm partials for 64 groups and three disjoint 64-float statistics slots ([mean, rstd] per group)
  if (c->norm_groups < 1 || c->norm_groups > 32)
    return mvb::set_error(MVB_ERR_ARG, "mbd: norm_groups %d out of range (1 .. 32)", c->norm_groups);
  int h = c->hidden;
  for (int i = 0; i < c->depth; ++i) {
    if (h % c->norm_groups) return mvb::set_error(MVB_ERR_ARG, "mbd: channels must be divisible by norm_groups");
    h = (int)(h * c->growth);
  }
  if (c->proc_bands < 2 || c->proc_bands > 64 || c->eq_bands < 2 || c->eq_bands > 64 || c->n_calls < 1 || c->n_calls > 1000)
    return mvb::set_error(MVB_ERR_ARG, "mbd: band / call counts out of range");
  for (int L : {c->proc_taps, c->eq_taps})
    if (L < 1 || fir_smem_bytes(L) > FIR_SMEM_MAX)
      return mvb::set_error(MVB_ERR_UNSUPPORTED, "mbd: filter length %d (1 .. %d taps)", L, (int)((FIR_SMEM_MAX / 4 - FIR_TT) / 3));
  if (c->max_samples < c->stride) return mvb::set_error(MVB_ERR_ARG, "mbd: max_samples");
  const int known = MVB_MBD_CUDA_CORES | MVB_MBD_ONE_STREAM;
  if (c->options & ~known) return mvb::set_error(MVB_ERR_ARG, "mbd: options: undefined bits 0x%x", (unsigned)(c->options & ~known));
  return MVB_OK;
}
static int mbd_per_model(const mvb_mbd_config* c) { return c->depth * (3 + 8 * c->res_blocks + 1) + 2 + c->depth * (8 * c->res_blocks + 3) + 2; }

// Convolutions of one band model in tensor order: fn(tensor index relative to the model, Cin, Cout, K, transposed)
template <class F>
static void mbd_for_each_conv(const mvb_mbd_config* c, F fn) {
  std::vector<int> ch;
  int h = c->hidden;
  for (int i = 0; i < c->depth; ++i) { ch.push_back(h); h = (int)(h * c->growth); }
  int ti = 0, cin = c->chin;
  for (int i = 0; i < c->depth; ++i) {
    fn(ti, cin, ch[i], c->kernel, 0);
    ti += 3;
    for (int j = 0; j < c->res_blocks; ++j) { fn(ti + 8 * j + 2, ch[i], ch[i], 3, 0); fn(ti + 8 * j + 6, ch[i], ch[i], 3, 0); }
    ti += 8 * c->res_blocks + 1;
    cin = ch[i];
  }
  ti += 2;
  for (int i = 0; i < c->depth; ++i) {
    const int lvl = c->depth - 1 - i;
    for (int j = 0; j < c->res_blocks; ++j) { fn(ti + 8 * j + 2, ch[lvl], ch[lvl], 3, 0); fn(ti + 8 * j + 6, ch[lvl], ch[lvl], 3, 0); }
    ti += 8 * c->res_blocks;
    fn(ti + 2, ch[lvl], lvl == 0 ? c->chin : ch[lvl - 1], c->kernel, 1);
    ti += 3;
  }
}
// Input widths >= 32 take the tensor-core path; the time-major copy and the packed taps are zero-padded to a multiple of 64 channels
static bool mbd_tc_eligible(int cin) { return cin >= 32; }
static int mbd_tc_cpad(int cin) { return (cin + 63) / 64 * 64; }
static MbdWs mbd_layout(const mvb_mbd_config* c) {
  MbdWs L{};
  WsBump ws;
  const size_t T = c->max_samples;
  L.cur = ws.take(T * 4); L.est = ws.take(T * 4); L.noise = ws.take(T * 4); L.wav = ws.take(T * 4);
  int h = c->hidden;
  size_t tl = T, big = 0;
  std::vector<size_t> lev;
  for (int i = 0; i < c->depth; ++i) {
    tl = (tl + c->stride - 1) / c->stride;
    lev.push_back((size_t)h * tl);
    big = big > (size_t)h * tl ? big : (size_t)h * tl;
    h = (int)(h * c->growth);
  }
  // the transposed convolutions write (stride x longer, growth x narrower) tensors: size the temporaries for the widest case
  size_t tmpsz = big * (size_t)(c->stride > c->growth ? c->stride / (c->growth > 1 ? c->growth : 1) + 1 : 2);
  if (tmpsz < T + 64) tmpsz = T + 64;
  L.cond = ws.take((size_t)(h / (int)c->growth) * (c->max_samples / 320 + 8) * 4);
  L.gn = ws.take(4096);
  L.gn_part = ws.take((size_t)64 * GN_SPLIT * 16);
  L.stdv = ws.take(4096);
  const int fb = (c->eq_bands > c->proc_bands ? c->eq_bands : c->proc_bands);
  L.low = ws.take((size_t)2 * fb * T * 4);
  for (int i = 0; i < c->depth; ++i) L.skip[i] = ws.take(lev[i] * 4);
  for (int i = 0; i < 3; ++i) L.tmp[i] = ws.take(tmpsz * 4);
  // time-major bf16 copies of one layer input (hi / lo) and the packed bf16 taps of every tensor-core convolution
  const size_t xt = (big * 2 + (size_t)h * (c->stride + 32)) * 2;   // (x2: widths below 64 are padded to 64 columns)
  L.xt_hi = ws.take(xt);
  L.xt_lo = ws.take(xt);
  WsBump wp;   // the packed taps of one band model
  L.tc = !(c->options & MVB_MBD_CUDA_CORES);
  if (L.tc)
    mbd_for_each_conv(c, [&](int, int cin, int cout, int k, int) {
      if (mbd_tc_eligible(cin)) wp.take((size_t)k * cout * mbd_tc_cpad(cin) * 2);
    });
  L.blk = (ws.end + 4095) / 4096 * 4096;
  // The band models are independent until their outputs are summed: each runs on its own stream with its own activation
  // block, so the many sub-wave kernels of one UNet (96-CTA convolutions, 4-CTA reductions) overlap with the other models'.
  L.n_blk = (!(c->options & MVB_MBD_ONE_STREAM) && c->n_models > 1) ? c->n_models : 1;
  L.wpack = L.blk * L.n_blk;
  L.total = L.wpack + wp.end * c->n_models + 256;
  return L;
}

extern "C" size_t mvb_mbd_workspace_bytes(const mvb_mbd_config* c) {
  if (mbd_validate(c)) return 0;
  return mbd_layout(c).total;
}

extern "C" int mvb_mbd_create(const mvb_mbd_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets, void* d_ws,
                              mvb_mbd** out) {
  if (int e = mbd_validate(cfg)) return e;
  if (!d_arena || !offsets || !d_ws || !out) return mvb::set_error(MVB_ERR_ARG, "null pointer argument");
  const int per_model = mbd_per_model(cfg), n_off = cfg->n_models * per_model + 3;
  if (int e = check_offsets(offsets, n_off, arena_bytes, "mbd: tensor offset")) return e;
  Building<mvb_mbd> hb(new mvb_mbd(), mvb_mbd_destroy);
  mvb_mbd* h = hb.get();
  h->cfg = *cfg;
  h->arena = reinterpret_cast<const char*>(d_arena);
  h->per_model = per_model;
  h->off.assign(offsets, offsets + n_off);
  h->ws = reinterpret_cast<char*>(d_ws);
  int c = cfg->hidden;
  for (int i = 0; i < cfg->depth; ++i) { h->ch.push_back(c); c = (int)(c * cfg->growth); }
  h->L = mbd_layout(cfg);
  const MbdWs& L = h->L;
  h->base = h->ws;
  if (L.n_blk > 1) {
    bool ok_s = cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; i < L.n_blk && ok_s; ++i)
      ok_s = cudaStreamCreateWithFlags(&h->st[i], cudaStreamNonBlocking) == cudaSuccess &&
             cudaEventCreateWithFlags(&h->ev_join[i], cudaEventDisableTiming) == cudaSuccess;
    if (!ok_s) return mvb::set_error(MVB_ERR_CUDA, "mbd: stream / event creation failed");
  }
  // tensor-core path: repack the taps of every eligible convolution to bf16 [tap][Cout][Cin] and build their A maps
  h->tc_of.assign(n_off, -1);
  if (L.tc && encode_tiled_fn()) {
    WsBump wo;
    bool ok = true;
    for (int m = 0; m < cfg->n_models && ok; ++m)
      mbd_for_each_conv(cfg, [&](int ti, int cin, int cout, int k, int tr) {
        if (!ok || !mbd_tc_eligible(cin)) return;
        const int gi = m * h->per_model + ti;
        const int cp = mbd_tc_cpad(cin);
        __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(h->ws + L.wpack + wo.take((size_t)k * cout * cp * 2));
        k_mbd_pack_w<<<GRID_STRIDE_CTAS * 4, 256>>>(h->w(gi), cout, cin, cp, k, tr, dst);
        mvb_mbd::TcW w{};
        w.Cin = cin; w.Cout = cout; w.K = k;
        ok = ok && make_tmap_bf16_3d(&w.tmA, dst, (uint64_t)cp, (uint64_t)cout, (uint64_t)k, (uint64_t)cout * cp * 2, 128);
        h->tc_of[gi] = (int)h->tcw.size();
        h->tcw.push_back(w);
      });
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_mbd_tc_conv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM);
    if (!ok || e != cudaSuccess)
      return mvb::set_error(MVB_ERR_CUDA, "mbd: tensor-core weight repack failed (%s)", ok ? cudaGetErrorString(e) : "tensor map");
  }
  *out = hb.release();
  return MVB_OK;
}
extern "C" int mvb_mbd_destroy(mvb_mbd* h) {
  if (h) {
    for (int i = 0; i < 8; ++i) {
      if (h->st[i]) cudaStreamDestroy(h->st[i]);
      if (h->ev_join[i]) cudaEventDestroy(h->ev_join[i]);
    }
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  }
  delete h;
  return MVB_OK;
}

static int launch_conv(cudaStream_t s, const ConvP& p, int K, int stride) {
  if (K == 3 && stride == 1) k_mbd_conv<3, 1, 4><<<dim3((p.Tout + 255) / 256, (p.Cout + 31) / 32), 256, 0, s>>>(p);
  else if (K == 1 && stride == 1) k_mbd_conv<1, 1, 4><<<dim3((p.Tout + 255) / 256, (p.Cout + 31) / 32), 256, 0, s>>>(p);
  else if (K == 8 && stride == 4) k_mbd_conv<8, 4, 1><<<dim3((p.Tout + 63) / 64, (p.Cout + 31) / 32), 256, 0, s>>>(p);
  else if (K == 4 && stride == 2) k_mbd_conv<4, 2, 2><<<dim3((p.Tout + 127) / 128, (p.Cout + 31) / 32), 256, 0, s>>>(p);
  else return mvb::set_error(MVB_ERR_UNSUPPORTED, "mbd: conv (k=%d, s=%d)", K, stride);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}
// part: room for groups x GN_SPLIT fp64 (sum, sum of squares) pairs
static int gn_stats(cudaStream_t s, double* part, const float* x, int C, int T, int groups, float eps, float* stats) {
  const size_t n = (size_t)(C / groups) * T;
  k_gn_partial<<<dim3(groups, GN_SPLIT), 256, 0, s>>>(x, n, part);
  k_gn_final<<<groups, 32, 0, s>>>(part, groups, (double)n, eps, stats);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

// One convolution on the tensor cores (mbd_tc.cuh).  kind 0: Conv1d stride 1 ('same', pad = dil * (K - 1) / 2);
// 1: Conv1d(K = 2s, stride s, pad s/2) over the right-padded input; 2: ConvTranspose1d(K = 2s, stride s, pad s/2).
// tmA: the taps packed by k_mbd_pack_w; hi / lo: room for the time-major copy of the input (Tpad x Cp bf16 each).
static int conv_tc(cudaStream_t s, const ConvP& p, const CUtensorMap& tmA, __nv_bfloat16* hi, __nv_bfloat16* lo, int kind, int K,
                   int stride) {
  const int Tpad = kind == 1 ? (p.Tin + stride - 1) / stride * stride : p.Tin;
  const int Cp = mbd_tc_cpad(p.Cin);
  k_mbd_prep_t<<<dim3((Tpad + 31) / 32, Cp / 64), 256, 0, s>>>(p.x, p.Cin, Cp, p.Tin, Tpad, p.gn_stats, p.gn_w, p.gn_b,
                                                              p.gn_stats ? p.Cin / p.groups : 1, hi, lo);
  MVB_CK(cudaGetLastError());
  const uint64_t rows = kind == 1 ? Tpad / stride : p.Tin, cols = kind == 1 ? (uint64_t)stride * Cp : Cp;
  CUtensorMap tBhi, tBlo;
  if (!make_tmap_bf16(&tBhi, hi, rows, cols, 128) || !make_tmap_bf16(&tBlo, lo, rows, cols, 128))
    return mvb::set_error(MVB_ERR_CUDA, "mbd: activation tensor map");
  TcConvP q{};
  q.Cin = Cp; q.M = p.Cout; q.out = p.y; q.ldo = p.Tout; q.bias = p.bias; q.emb = p.emb; q.resid = p.resid;
  q.Ncols = kind == 2 ? p.Tin : p.Tout;
  q.ostride = kind == 2 ? stride : 1;
  TcTaps& t = q.taps;
  if (kind == 0) {
    t.n_ph = 1; t.n_slots = K;
    for (int k = 0; k < K; ++k) { t.a_z[0][k] = k; t.b_shift[0][k] = k * p.dil - p.pad; t.b_col[0][k] = 0; }
  } else if (kind == 1) {
    t.n_ph = 1; t.n_slots = K;
    for (int k = 0; k < K; ++k) {
      const int o = k - p.pad;
      const int qd = o >= 0 ? o / stride : -((-o + stride - 1) / stride);
      t.a_z[0][k] = k; t.b_shift[0][k] = qd; t.b_col[0][k] = (o - qd * stride) * Cp;
    }
  } else {
    t.n_ph = stride; t.n_slots = 2;
    for (int ph = 0; ph < stride; ++ph) {
      const int e = ph + p.pad;
      t.a_z[ph][0] = e % stride;          t.b_shift[ph][0] = e / stride;     t.b_col[ph][0] = 0;
      t.a_z[ph][1] = e % stride + stride; t.b_shift[ph][1] = e / stride - 1; t.b_col[ph][1] = 0;
    }
  }
  const int n_cot = (p.Cout + 127) / 128;
  k_mbd_tc_conv<<<dim3(t.n_ph * n_cot, (q.Ncols + 127) / 128), TC_THREADS, TC_SMEM, s>>>(tmA, tBhi, tBlo, q);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}
static int launch_conv_tc(mvb_mbd* h, cudaStream_t s, const ConvP& p, int widx, int kind, int K, int stride) {
  const MbdWs& L = h->L;
  return conv_tc(s, p, h->tcw[h->tc_of[widx]].tmA, reinterpret_cast<__nv_bfloat16*>(h->base + L.xt_hi),
                 reinterpret_cast<__nv_bfloat16*>(h->base + L.xt_lo), kind, K, stride);
}

// ResBlock (unet.py): x + conv2(relu(norm2(conv1(relu(norm1(x)))))), kernel 3, dilation 2^j; `emb` is added to the block output
static int res_block(mvb_mbd* h, cudaStream_t s, int base, int C, int T, int dil, const float* x, float* tmp, float* out, float* stats,
                     const float* emb) {
  ConvP p{};
  double* part = reinterpret_cast<double*>(h->base + h->L.gn_part);
  if (int e = gn_stats(s, part, x, C, T, h->cfg.norm_groups, GN_EPS, stats)) return e;
  p.x = x; p.Cin = C; p.Tin = T; p.w = h->w(base + 2); p.bias = h->w(base + 3); p.y = tmp; p.Cout = C; p.Tout = T; p.dil = dil; p.pad = dil;
  p.gn_stats = stats; p.gn_w = h->w(base); p.gn_b = h->w(base + 1); p.groups = h->cfg.norm_groups;
  if (int e = h->tc_of[base + 2] >= 0 ? launch_conv_tc(h, s, p, base + 2, 0, 3, 1) : launch_conv(s, p, 3, 1)) return e;
  if (int e = gn_stats(s, part, tmp, C, T, h->cfg.norm_groups, GN_EPS, stats + 64)) return e;
  p.x = tmp; p.w = h->w(base + 6); p.bias = h->w(base + 7); p.y = out; p.gn_stats = stats + 64; p.gn_w = h->w(base + 4); p.gn_b = h->w(base + 5);
  p.resid = x; p.emb = emb;
  return h->tc_of[base + 6] >= 0 ? launch_conv_tc(h, s, p, base + 6, 0, 3, 1) : launch_conv(s, p, 3, 1);
}

// DiffusionUnet.forward (unet.py) for band model m: est <- model(cur, step, cond)
static int unet_forward(mvb_mbd* h, cudaStream_t s, int m, int step, const float* cur, int T, const float* d_cond, int Tf, float* est) {
  const mvb_mbd_config& c = h->cfg;
  const MbdWs& L = h->L;
  float* stats = reinterpret_cast<float*>(h->base + L.gn);
  double* part = reinterpret_cast<double*>(h->base + L.gn_part);
  float* tmp[3] = {reinterpret_cast<float*>(h->base + L.tmp[0]), reinterpret_cast<float*>(h->base + L.tmp[1]), reinterpret_cast<float*>(h->base + L.tmp[2])};
  const int pad_k = (c.kernel - c.stride) / 2, G = c.norm_groups;
  int ti = m * h->per_model;
  const float* x = cur;
  int Cin = 1, Tl = T;
  std::vector<int> Ts;
  for (int i = 0; i < c.depth; ++i) {
    const int C = h->ch[i];
    const int To = (Tl + c.stride - 1) / c.stride;      // right zero-padding to a multiple of the stride, then k = 2s, p = s/2
    ConvP p{};
    p.x = x; p.Cin = Cin; p.Tin = Tl; p.w = h->w(ti); p.y = tmp[0]; p.Cout = C; p.Tout = To; p.dil = 1; p.pad = pad_k;
    if (int e = h->tc_of[ti] >= 0 ? launch_conv_tc(h, s, p, ti, 1, c.kernel, c.stride) : launch_conv(s, p, c.kernel, c.stride)) return e;
    // norm -> relu -> res_blocks: the first ResBlock input is relu(GN(conv)); materialise it (it is also the residual)
    if (int e = gn_stats(s, part, tmp[0], C, To, G, GN_EPS, stats + 128)) return e;
    k_gn_relu_inplace<<<GRID_STRIDE_CTAS * 4, 256, 0, s>>>(tmp[0], C, To, C / G, stats + 128, h->w(ti + 1), h->w(ti + 2));
    MVB_CK(cudaGetLastError());
    ti += 3;
    float* a = tmp[0];
    float* b = tmp[1];
    float* skip = reinterpret_cast<float*>(h->base + L.skip[i]);
    const float* emb = nullptr;
    for (int j = 0; j < c.res_blocks; ++j) {
      const bool last = j == c.res_blocks - 1;
      if (last && (i == 0 || c.emb_all_layers)) emb = h->w(ti + 8 * c.res_blocks) + (size_t)step * C;
      float* dst = last ? skip : b;
      if (int e = res_block(h, s, ti + 8 * j, C, To, 1 << j, a, tmp[2], dst, stats, last ? emb : nullptr)) return e;
      if (!last) { float* t = a; a = b; b = t; }
    }
    ti += 8 * c.res_blocks + 1;
    x = skip; Cin = C; Tl = To;
    Ts.push_back(To);
  }
  // condition in the bottleneck: z += nearest-interpolate(conv_codec(cond))
  const int Cb = h->ch[c.depth - 1];
  float* z = tmp[0];
  {
    float* cemb = reinterpret_cast<float*>(h->base + L.cond);
    ConvP p{};
    p.x = d_cond; p.Cin = c.codec_dim; p.Tin = Tf; p.w = h->w(ti); p.bias = h->w(ti + 1); p.y = cemb; p.Cout = Cb; p.Tout = Tf; p.dil = 1; p.pad = 0;
    if (int e = launch_conv(s, p, 1, 1)) return e;
    MVB_CK(cudaMemcpyAsync(z, x, sizeof(float) * (size_t)Cb * Tl, cudaMemcpyDeviceToDevice, s));
    k_add_interp<<<GRID_STRIDE_CTAS * 2, 256, 0, s>>>(z, Tl, cemb, Tf, Cb);
    MVB_CK(cudaGetLastError());
    ti += 2;
  }
  // decoders (deepest first): z = crop(z) + skip; res_blocks; norm; relu; convtr.  Three temporaries rotate: z lives in
  // tmp[zi]; the skip sum goes to tmp[zi+1]; tmp[zi+2] is the ResBlock scratch and then receives the transposed convolution.
  int Tz = Tl, zi = 0;
  for (int i = 0; i < c.depth; ++i) {
    const int lvl = c.depth - 1 - i, C = h->ch[lvl], Tsk = Ts[lvl];
    const float* skip = reinterpret_cast<const float*>(h->base + L.skip[lvl]);
    float* a = tmp[(zi + 1) % 3];
    float* b = tmp[zi];                   // free once the skip sum has been formed
    float* scratch = tmp[(zi + 2) % 3];
    k_add_crop<<<GRID_STRIDE_CTAS * 2, 256, 0, s>>>(z, Tz, skip, Tsk, C, a);
    MVB_CK(cudaGetLastError());
    for (int j = 0; j < c.res_blocks; ++j) {
      if (int e = res_block(h, s, ti + 8 * j, C, Tsk, 1 << j, a, scratch, b, stats, nullptr)) return e;
      float* t = a; a = b; b = t;
    }
    ti += 8 * c.res_blocks;
    if (int e = gn_stats(s, part, a, C, Tsk, G, GN_EPS, stats + 128)) return e;
    const int Cout = lvl == 0 ? 1 : h->ch[lvl - 1];
    const int To = Tsk * c.stride;
    ConvP p{};
    p.x = a; p.Cin = C; p.Tin = Tsk; p.w = h->w(ti + 2); p.y = scratch; p.Cout = Cout; p.Tout = To; p.pad = pad_k;
    p.gn_stats = stats + 128; p.gn_w = h->w(ti); p.gn_b = h->w(ti + 1); p.groups = G;
    if (h->tc_of[ti + 2] >= 0) {
      if (int e = launch_conv_tc(h, s, p, ti + 2, 2, c.kernel, c.stride)) return e;
    } else if (c.stride == 4) k_mbd_convtr<4><<<dim3((To + 255) / 256, (Cout + 31) / 32), 256, 0, s>>>(p);
    else k_mbd_convtr<2><<<dim3((To + 255) / 256, (Cout + 31) / 32), 256, 0, s>>>(p);
    MVB_CK(cudaGetLastError());
    ti += 3;
    z = scratch; Tz = To; zi = (zi + 2) % 3;
  }
  // crop to the input length
  MVB_CK(cudaMemcpyAsync(est, z, sizeof(float) * (size_t)T, cudaMemcpyDeviceToDevice, s));
  return MVB_OK;
}

// The n_bands - 1 low-passed copies of x [T] through bank [n_bands - 1, L] into low [n_bands - 1, T].  k_fir_bank is opted
// into 64 KB of dynamic shared memory (every bank up to 55 bands at 24 kHz), and into more, up to the device's opt-in
// maximum, the first time a longer filter runs on the device.
static int split_lows(cudaStream_t s, const float* x, int T, int n_bands, const float* bank, int L, float* low) {
  const size_t smem = fir_smem_bytes(L);
  static size_t opted[64] = {};
  int dev = 0;
  MVB_CK(cudaGetDevice(&dev));
  size_t& cur = opted[dev >= 0 && dev < 64 ? dev : 0];
  if (cur == 0 || smem > cur) {
    const size_t want = smem > 64 * 1024 ? smem : 64 * 1024;
    int optin = 0;
    MVB_CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    if (want > (size_t)optin) return mvb::set_error(MVB_ERR_UNSUPPORTED, "mbd: filter length %d needs %zu B of shared memory", L, smem);
    MVB_CK(cudaFuncSetAttribute(k_fir_bank, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)want));
    cur = want;
  }
  k_fir_bank<<<dim3((T + FIR_TT - 1) / FIR_TT, (n_bands - 1 + 1) / 2), 256, smem, s>>>(x, T, bank, L, n_bands - 1, low);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

// The shape checks of one UNet call, made before anything is enqueued.  The codec condition is projected into L.cond,
// which holds max_samples / 320 + 8 frames, and then interpolated onto the bottleneck, which may downsample it at most
// 2x (the restatement's assert): n_frames <= 2 Tl, Tl = n_samples divided depth times by the stride, rounded up.
static int mbd_check_shape(const mvb_mbd_config& c, int32_t n_frames, int32_t n_samples) {
  if (n_samples < 16 * c.stride || n_samples > c.max_samples) return mvb::set_error(MVB_ERR_ARG, "mbd: n_samples %d out of range", n_samples);
  if (n_frames < 1) return mvb::set_error(MVB_ERR_ARG, "mbd: n_frames %d", n_frames);
  const int cap = c.max_samples / 320 + 8;
  if (n_frames > cap)
    return mvb::set_error(MVB_ERR_ARG, "mbd: n_frames %d exceeds the condition capacity %d (max_samples %d)", n_frames, cap, c.max_samples);
  int tl = n_samples;
  for (int i = 0; i < c.depth; ++i) tl = (tl + c.stride - 1) / c.stride;
  if (n_frames > 2 * tl)
    return mvb::set_error(MVB_ERR_ARG, "mbd: n_frames %d is more than twice the bottleneck length %d of %d samples", n_frames, tl,
                          n_samples);
  return MVB_OK;
}

// Every shape check (mbd_check_shape: n_samples, and n_frames against the L.cond capacity and the bottleneck) runs before
// the first copy, launch or stream fork.
extern "C" int mvb_mbd_tokens_to_wav(mvb_mbd* h, const float* d_cond, int32_t n_frames, const float* d_wav_encodec, int32_t n_samples,
                                     const float* d_noise, uint64_t seed, float* d_wav_out, void* stream) {
  if (!h || !d_cond || !d_wav_encodec || !d_wav_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  const mvb_mbd_config& c = h->cfg;
  if (int e = mbd_check_shape(c, n_frames, n_samples)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  const MbdWs& L = h->L;
  const int T = n_samples;
  const bool multi = L.n_blk > 1;
  h->base = h->ws;
  float* wav = reinterpret_cast<float*>(h->ws + L.wav);      // block 0: the sum over the band models, then the re-EQ input
  float* low = reinterpret_cast<float*>(h->ws + L.low);
  float* stdv = reinterpret_cast<float*>(h->ws + L.stdv);
  const int g0 = c.n_models * h->per_model;          // globals: processor bank, eq bank, schedule table
  const float* sched = h->w(g0 + 2);                 // [n_calls][4] = a, b, sigma, step
  std::vector<float> hs((size_t)c.n_calls * 4);
  MVB_CK(cudaMemcpyAsync(hs.data(), sched, sizeof(float) * hs.size(), cudaMemcpyDeviceToHost, s));
  MVB_CK(cudaStreamSynchronize(s));
  if (!multi) MVB_CK(cudaMemsetAsync(wav, 0, sizeof(float) * T, s));
  if (multi) MVB_CK(cudaEventRecord(h->ev_fork, s));
  int rc = MVB_OK;
  for (int m = 0; m < c.n_models && rc == MVB_OK; ++m) {
    cudaStream_t sm = multi ? h->st[m] : s;
    h->base = h->ws + (multi ? (size_t)m * L.blk : 0);
    if (multi) MVB_CK(cudaStreamWaitEvent(sm, h->ev_fork, 0));
    float* cur = reinterpret_cast<float*>(h->base + L.cur);
    float* est = reinterpret_cast<float*>(h->base + L.est);
    float* nz = reinterpret_cast<float*>(h->base + L.noise);
    float* wav_m = reinterpret_cast<float*>(h->base + L.wav);
    float* low_m = reinterpret_cast<float*>(h->base + L.low);
    // initial = randn * noise_scale
    const float* n0 = d_noise ? d_noise + ((size_t)m * c.n_calls) * T : nz;
    if (!d_noise) { k_randn<<<GRID_STRIDE_CTAS, 256, 0, sm>>>(nz, T, seed, (unsigned)(m * 1024)); MVB_CK(cudaGetLastError()); }
    k_scale_copy<<<GRID_STRIDE_CTAS, 256, 0, sm>>>(n0, c.noise_scale, cur, T);
    MVB_CK(cudaGetLastError());
    for (int i = 0; i < c.n_calls; ++i) {
      const float a = hs[4 * i], b = hs[4 * i + 1], sigma = hs[4 * i + 2];
      const int step = (int)hs[4 * i + 3];
      if ((rc = unet_forward(h, sm, m, step, cur, T, d_cond, n_frames, est)) != MVB_OK) break;
      const float* ni = nullptr;
      if (sigma > 0.f) {
        if (d_noise) ni = d_noise + ((size_t)m * c.n_calls + i + 1) * T;      // row i + 1: the draw added after call i
        else { k_randn<<<GRID_STRIDE_CTAS, 256, 0, sm>>>(nz, T, seed, (unsigned)(m * 1024 + i + 1)); MVB_CK(cudaGetLastError()); ni = nz; }
      }
      k_sched_step<<<GRID_STRIDE_CTAS * 2, 256, 0, sm>>>(cur, est, ni, a, b, sigma, c.noise_scale, c.clip, T);
      MVB_CK(cudaGetLastError());
    }
    if (rc != MVB_OK) break;
    // MultiBandProcessor.return_sample: bands * (std / target_std) ** power_std + mean, summed; the band models' outputs are
    // added up in model order (one stream: accumulated in place; several streams: per-model buffers summed after the join)
    const int pb = m * h->per_model + h->per_model - 2;
    if ((rc = split_lows(sm, cur, T, c.proc_bands, h->w(g0), c.proc_taps, low_m)) != MVB_OK) break;
    k_band_mix<<<GRID_STRIDE_CTAS * 2, 256, 0, sm>>>(low_m, cur, T, c.proc_bands, h->w(pb), nullptr, h->w(pb + 1), wav_m, multi ? 0 : 1);
    MVB_CK(cudaGetLastError());
    if (multi) MVB_CK(cudaEventRecord(h->ev_join[m], sm));
  }
  h->base = h->ws;
  if (multi) {
    // always re-join the caller's stream, also on an error path, so no work is left running behind the caller's back
    for (int m = 0; m < c.n_models; ++m) MVB_CK(cudaStreamWaitEvent(s, h->ev_join[m], 0));   // (an event never recorded in this call is complete)
    if (rc == MVB_OK) {
      k_sum_blocks<<<GRID_STRIDE_CTAS * 2, 256, 0, s>>>(wav, L.blk / 4, c.n_models, T);
      MVB_CK(cudaGetLastError());
    }
  }
  if (rc != MVB_OK) return rc;
  // re_eq(wav, ref = wav_encodec, eq_bands): out = sum_b band_b(wav) * std(band_b(ref)) / std(band_b(wav))
  float* low_w = low;
  float* low_r = low + (size_t)c.eq_bands * T;
  if (int e = split_lows(s, wav, T, c.eq_bands, h->w(g0 + 1), c.eq_taps, low_w)) return e;
  if (int e = split_lows(s, d_wav_encodec, T, c.eq_bands, h->w(g0 + 1), c.eq_taps, low_r)) return e;
  k_band_std<<<c.eq_bands, 256, 0, s>>>(low_w, wav, T, c.eq_bands, stdv);
  MVB_CK(cudaGetLastError());
  k_band_std<<<c.eq_bands, 256, 0, s>>>(low_r, d_wav_encodec, T, c.eq_bands, stdv + 64);
  MVB_CK(cudaGetLastError());
  k_band_mix<<<GRID_STRIDE_CTAS * 2, 256, 0, s>>>(low_w, wav, T, c.eq_bands, stdv + 64, stdv, nullptr, d_wav_out, 0);
  MVB_CK(cudaGetLastError());
  return MVB_OK;
}

// Test hook: the unet_forward of tokens_to_wav for band model `model` at the step of schedule row `call`, in that model's
// activation block (block 0 under MVB_MBD_ONE_STREAM), on `stream`: d_est [n_samples] <- UNet(d_cur, step, d_cond).
// The shape checks of tokens_to_wav.  Synchronises `stream`.
extern "C" int mvb_mbd_unet_test(mvb_mbd* h, int32_t model, int32_t call, const float* d_cur, int32_t n_samples, const float* d_cond,
                                 int32_t n_frames, float* d_est, void* stream) {
  if (!h || !d_cur || !d_cond || !d_est) return mvb::set_error(MVB_ERR_ARG, "null argument");
  const mvb_mbd_config& c = h->cfg;
  if (model < 0 || model >= c.n_models || call < 0 || call >= c.n_calls)
    return mvb::set_error(MVB_ERR_ARG, "mvb_mbd_unet_test: model %d / call %d out of range", model, call);
  if (int e = mbd_check_shape(c, n_frames, n_samples)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  float row[4];
  MVB_CK(cudaMemcpyAsync(row, h->w(c.n_models * h->per_model + 2) + 4 * (size_t)call, sizeof(row), cudaMemcpyDeviceToHost, s));
  MVB_CK(cudaStreamSynchronize(s));
  h->base = h->ws + (h->L.n_blk > 1 ? (size_t)model * h->L.blk : 0);
  int rc = unet_forward(h, s, model, (int)row[3], d_cur, n_samples, d_cond, n_frames, d_est);
  h->base = h->ws;
  const cudaError_t e = cudaStreamSynchronize(s);
  if (rc == MVB_OK && e != cudaSuccess) rc = mvb::set_error(MVB_ERR_CUDA, "mvb_mbd_unet_test: %s", cudaGetErrorString(e));
  return rc;
}

// Test hook: one convolution of the kinds unet_forward runs, outside any mvb_mbd handle, with the taps packed by
// k_mbd_pack_w and the input prepared by k_mbd_prep_t exactly as in the engine (use_tc != 0), or through the CUDA-core
// kernels (use_tc == 0).  Buffers for the packed taps and the time-major input are allocated per call.  Synchronises `stream`.
extern "C" int mvb_mbd_conv_test(int32_t kind, const float* d_x, int32_t Cin, int32_t Tin, const float* d_w, int32_t Cout, int32_t K,
                                 int32_t stride, int32_t dil, int32_t pad, const float* d_gn_stats, const float* d_gn_w,
                                 const float* d_gn_b, int32_t groups, const float* d_bias, const float* d_emb, const float* d_resid,
                                 float* d_y, int32_t use_tc, void* stream) {
  if (!d_x || !d_w || !d_y) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (kind < 0 || kind > 2 || Cin < 1 || Cout < 1 || Tin < 1 || K < 1 || stride < 1 || dil < 1 || pad < 0)
    return mvb::set_error(MVB_ERR_ARG, "mvb_mbd_conv_test: bad shape");
  if (d_gn_stats && (!d_gn_w || !d_gn_b || groups < 1 || Cin % groups)) return mvb::set_error(MVB_ERR_ARG, "mvb_mbd_conv_test: GroupNorm");
  if ((kind == 0 && (stride != 1 || 2 * pad != dil * (K - 1))) || (kind != 0 && (K != 2 * stride || dil != 1)) ||
      (kind == 2 && (d_bias || d_emb || d_resid)))
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_mbd_conv_test: kind %d with K %d stride %d dil %d pad %d", kind, K, stride, dil, pad);
  cudaStream_t s = (cudaStream_t)stream;
  ConvP p{};
  p.x = d_x; p.Cin = Cin; p.Tin = Tin; p.w = d_w; p.bias = d_bias; p.y = d_y; p.Cout = Cout;
  p.Tout = kind == 0 ? Tin : kind == 1 ? (Tin + stride - 1) / stride : Tin * stride;
  p.dil = dil; p.pad = pad;
  p.gn_stats = d_gn_stats; p.gn_w = d_gn_w; p.gn_b = d_gn_b; p.groups = groups;
  p.resid = d_resid; p.emb = d_emb;
  if (!use_tc) {
    if (kind != 2) {
      if (int e = launch_conv(s, p, K, stride)) return e;
    } else if (stride == 4) k_mbd_convtr<4><<<dim3((p.Tout + 255) / 256, (Cout + 31) / 32), 256, 0, s>>>(p);
    else if (stride == 2) k_mbd_convtr<2><<<dim3((p.Tout + 255) / 256, (Cout + 31) / 32), 256, 0, s>>>(p);
    else return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_mbd_conv_test: transposed stride %d", stride);
    MVB_CK(cudaGetLastError());
    MVB_CK(cudaStreamSynchronize(s));
    return MVB_OK;
  }
  if ((kind != 2 && K > 8) || (kind == 2 && stride > 4)) return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_mbd_conv_test: too many taps");
  if (!encode_tiled_fn()) return mvb::set_error(MVB_ERR_CUDA, "mvb_mbd_conv_test: no cuTensorMapEncodeTiled");
  const int Cp = mbd_tc_cpad(Cin);
  const int Tpad = kind == 1 ? (Tin + stride - 1) / stride * stride : Tin;
  const size_t wbytes = (size_t)K * Cout * Cp * 2, xbytes = (size_t)Tpad * Cp * 2;
  WsBump ws;
  const size_t o_wp = ws.take(wbytes), o_hi = ws.take(xbytes), o_lo = ws.take(xbytes);
  char* buf = nullptr;
  MVB_CK(cudaMalloc(&buf, ws.end + 256));
  __nv_bfloat16* wp = reinterpret_cast<__nv_bfloat16*>(buf + o_wp);
  __nv_bfloat16* hi = reinterpret_cast<__nv_bfloat16*>(buf + o_hi);
  __nv_bfloat16* lo = reinterpret_cast<__nv_bfloat16*>(buf + o_lo);
  int rc = MVB_OK;
  cudaError_t e = cudaFuncSetAttribute(k_mbd_tc_conv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM);
  CUtensorMap tmA;
  if (e == cudaSuccess) {
    k_mbd_pack_w<<<GRID_STRIDE_CTAS * 4, 256, 0, s>>>(d_w, Cout, Cin, Cp, K, kind == 2 ? 1 : 0, wp);
    e = cudaGetLastError();
  }
  if (e != cudaSuccess) rc = mvb::set_error(MVB_ERR_CUDA, "mvb_mbd_conv_test: %s", cudaGetErrorString(e));
  else if (!make_tmap_bf16_3d(&tmA, wp, (uint64_t)Cp, (uint64_t)Cout, (uint64_t)K, (uint64_t)Cout * Cp * 2, 128))
    rc = mvb::set_error(MVB_ERR_CUDA, "mvb_mbd_conv_test: weight tensor map");
  else rc = conv_tc(s, p, tmA, hi, lo, kind, K, stride);
  e = cudaStreamSynchronize(s);    // (also on an error path: the buffer is freed only once nothing can still use it)
  if (rc == MVB_OK && e != cudaSuccess) rc = mvb::set_error(MVB_ERR_CUDA, "mvb_mbd_conv_test: %s", cudaGetErrorString(e));
  cudaFree(buf);
  return rc;
}

// Test hook: one launch of a non-convolution kernel of mvb_mbd_tokens_to_wav with the engine's launch configuration (for
// GroupNorm statistics and the FIR bank, through the engine's own gn_stats / split_lows).  Operands by op (see the header):
// a .. e inputs, out the output (in place for the ops that update a tensor), i0 .. i2 sizes, f0 .. f4 scalars.  The fp64
// GroupNorm partials are allocated per call.  Synchronises `stream`.
extern "C" int mvb_mbd_op_test(int32_t op, const float* d_a, const float* d_b, const float* d_c, const float* d_d, const float* d_e,
                               float* d_out, int32_t i0, int32_t i1, int32_t i2, float f0, float f1, float f2, float f3, float f4,
                               uint64_t seed, void* stream) {
  if (!d_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  auto need = [](bool ok) { return ok ? MVB_OK : mvb::set_error(MVB_ERR_ARG, "mvb_mbd_op_test: bad operands"); };
  switch (op) {
    case 0: {   // GroupNorm statistics of a [i0, i1] into out [i2][mean, rstd], eps f0
      if (int e = need(d_a && i0 >= 1 && i1 >= 1 && i2 >= 1 && i2 <= 64 && i0 % i2 == 0)) return e;
      double* part = nullptr;
      MVB_CK(cudaMalloc(&part, sizeof(double) * 2 * GN_SPLIT * i2));
      int rc = gn_stats(s, part, d_a, i0, i1, i2, f0, d_out);
      const cudaError_t ce = cudaStreamSynchronize(s);    // (also on an error path: freed only once nothing can use it)
      cudaFree(part);
      if (rc == MVB_OK && ce != cudaSuccess) rc = mvb::set_error(MVB_ERR_CUDA, "mvb_mbd_op_test: %s", cudaGetErrorString(ce));
      return rc;
    }
    case 1:     // out [i0, i1] <- relu(GroupNorm(out)) in place, i2 groups, statistics a, gain b, bias c
      if (int e = need(d_a && d_b && d_c && i0 >= 1 && i1 >= 1 && i2 >= 1 && i0 % i2 == 0)) return e;
      k_gn_relu_inplace<<<GRID_STRIDE_CTAS * 4, 256, 0, s>>>(d_out, i0, i1, i0 / i2, d_a, d_b, d_c);
      break;
    case 2:     // out [i0, i1] <- the i0 low-passed copies of a [i1] through bank b [i0, i2]
      if (int e = need(d_a && d_b && i0 >= 1 && i0 <= 63 && i1 >= 1 && i2 >= 1)) return e;
      if (int e = split_lows(s, d_a, i1, i0 + 1, d_b, i2, d_out)) return e;
      break;
    case 3:     // out [i0] <- unbiased std of the i0 bands of x = b [i1] given its low-passed copies a [i0 - 1, i1]
      if (int e = need(d_a && d_b && i0 >= 2 && i0 <= 64 && i1 >= 2)) return e;
      k_band_std<<<i0, 256, 0, s>>>(d_a, d_b, i1, i0, d_out);
      break;
    case 4:     // out [i1] (+)= sum_b band_b * scale_b + shift_b with scale = c / d (d may be null), shift e (may be null);
                // i2 != 0 accumulates
      if (int e = need(d_a && d_b && d_c && i0 >= 2 && i0 <= 64 && i1 >= 1)) return e;
      k_band_mix<<<GRID_STRIDE_CTAS * 2, 256, 0, s>>>(d_a, d_b, i1, i0, d_c, d_d, d_e, d_out, i2);
      break;
    case 5:     // out [i0, i1] += nearest-interpolated a [i0, i2]
      if (int e = need(d_a && i0 >= 1 && i1 >= 1 && i2 >= 1)) return e;
      k_add_interp<<<GRID_STRIDE_CTAS * 2, 256, 0, s>>>(d_out, i1, d_a, i2, i0);
      break;
    case 6:     // out [i0, i1] <- a [i0, i2] cropped to i1 + b [i0, i1]
      if (int e = need(d_a && d_b && i0 >= 1 && i1 >= 1 && i2 >= i1)) return e;
      k_add_crop<<<GRID_STRIDE_CTAS * 2, 256, 0, s>>>(d_a, i2, d_b, i1, i0, d_out);
      break;
    case 7:     // one schedule step on out [i1]: estimate a, noise b (may be null when sigma <= 0), a f0, b f1, sigma f2,
                // noise scale f3, clip f4
      if (int e = need(d_a && i1 >= 1)) return e;
      k_sched_step<<<GRID_STRIDE_CTAS * 2, 256, 0, s>>>(d_out, d_a, d_b, f0, f1, f2, f3, f4, i1);
      break;
    case 8:     // out [i1] <- standard-normal draws of Philox stream i2 under seed
      if (int e = need(i1 >= 1)) return e;
      k_randn<<<GRID_STRIDE_CTAS, 256, 0, s>>>(d_out, i1, seed, (unsigned)i2);
      break;
    case 9:     // out [i1] <- sum of the i0 blocks out + m i2 (m = 0 .. i0 - 1), in block order
      if (int e = need(i0 >= 1 && i1 >= 1 && (i0 == 1 || i2 >= i1))) return e;
      k_sum_blocks<<<GRID_STRIDE_CTAS * 2, 256, 0, s>>>(d_out, (size_t)i2, i0, i1);
      break;
    case 10:    // out [i1] <- a * f0
      if (int e = need(d_a && i1 >= 1)) return e;
      k_scale_copy<<<GRID_STRIDE_CTAS, 256, 0, s>>>(d_a, f0, d_out, i1);
      break;
    default:
      return mvb::set_error(MVB_ERR_ARG, "mvb_mbd_op_test: op %d", op);
  }
  MVB_CK(cudaGetLastError());
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}
