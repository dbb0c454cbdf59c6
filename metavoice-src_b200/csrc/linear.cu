// Standalone tensor-core linear operator (C ABI): y[R, M] (+)= f(x)[R, K] . W[M, K]^T with W in bf16.
// Used by the parity tests to validate the TMA / mma.sync path in isolation and by the stage-2 model.
#include <cstdio>
#include <string>

#include "../../include/mvb200.h"
#include "umma_host.cuh"

using namespace mvb;

extern "C" const char* mvb_last_error(void);
namespace mvb { int set_error(int code, const char* fmt, ...); }

#define LCK(expr)                                                                                   \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) {                                                                        \
      rc = mvb::set_error(MVB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      goto done;                                                                                    \
    }                                                                                               \
  } while (0)

namespace {

// Fields of GemmP the caller chooses for one epilogue: the output and, for G_QKV, the KV-cache scatter.
struct EpiArgs {
  float* out; int ldo;
  void* kcache; void* vcache; const int* row_cache; const int* row_pos;
  int H, S_max, D, kv_fp32;
};

// One k_umma_gemm launch with the RMSNorm / hi-lo prologue of k_prep_b, for any epilogue (W3 is the second weight of
// G_SWIGLU).  Synchronises `s`.
int run_gemm(int epi, const void* d_W, const void* d_W3, int M, int K, const float* d_x, int ldx, int R, const void* d_gain,
             float eps, int split_lo, int ksplit_override, const EpiArgs& ea, cudaStream_t s) {
  int rc = MVB_OK;
  const bool swiglu = epi == G_SWIGLU;
  const int Rpad = (R + 15) / 16 * 16;
  const int NB = Rpad * (split_lo ? 2 : 1);
  int n_sm = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  GemmPlan g = plan_gemm(M, K, NB, swiglu, n_sm);
  if (ksplit_override > 0) {
    // every split of a tile waits for its siblings inside the kernel: all tiles x ksplit CTAs must be co-resident
    const int cap = n_sm / g.tiles > 0 ? n_sm / g.tiles : 1;
    g.ksplit = ksplit_override < cap ? ksplit_override : cap;
    if (g.tiles > 128) g.ksplit = 1;
    g.scratch_floats = (size_t)g.tiles * g.ksplit * (swiglu ? 2 : 1) * NB * 128;
  }
  // Scratch buffers are cached per device and only ever grow (no allocation on the steady-state path; this standalone
  // operator has no caller-provided workspace, unlike the engine handles).
  struct Cache { void* p = nullptr; size_t cap = 0; };
  static Cache cB[16], cS[16], cT[16];
  auto ensure = [&](Cache& c, size_t bytes) -> cudaError_t {
    if (c.cap >= bytes) return cudaSuccess;
    if (c.p) cudaFree(c.p);
    c.p = nullptr; c.cap = 0;
    cudaError_t e = cudaMalloc(&c.p, bytes);
    if (e == cudaSuccess) c.cap = bytes;
    return e;
  };
  if (dev < 0 || dev >= 16) return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_linear: device index %d", dev);
  __nv_bfloat16* B = nullptr;
  float* scratch = nullptr;
  unsigned* tickets = nullptr;
  CUtensorMap tA, tA3, tB;
  GemmP p{};
  LCK(ensure(cB[dev], (size_t)NB * K * 2));
  LCK(ensure(cS[dev], sizeof(float) * (g.scratch_floats ? g.scratch_floats : 1)));
  LCK(ensure(cT[dev], sizeof(unsigned) * 256));
  B = reinterpret_cast<__nv_bfloat16*>(cB[dev].p);
  scratch = reinterpret_cast<float*>(cS[dev].p);
  tickets = reinterpret_cast<unsigned*>(cT[dev].p);
  LCK(cudaMemsetAsync(B, 0, (size_t)NB * K * 2, s));
  LCK(cudaMemsetAsync(tickets, 0, sizeof(unsigned) * 256, s));
  if (!make_tmap_bf16(&tA, d_W, (uint64_t)M, (uint64_t)K, 128) ||
      (swiglu && !make_tmap_bf16(&tA3, d_W3, (uint64_t)M, (uint64_t)K, 128)) ||
      !make_tmap_bf16(&tB, B, (uint64_t)NB, (uint64_t)K, (uint32_t)NB)) {
    rc = mvb::set_error(MVB_ERR_CUDA, "cuTensorMapEncodeTiled failed");
    goto done;
  }
  k_prep_b<<<Rpad, 256, 0, s>>>(d_x, ldx, reinterpret_cast<const __nv_bfloat16*>(d_gain), eps, K, Rpad, R, split_lo ? 1 : 0, B);
  LCK(cudaGetLastError());
  p.M = M; p.K = K; p.NB = NB; p.Rpad = Rpad; p.R = R; p.split_lo = split_lo ? 1 : 0;
  p.scratch = scratch; p.tickets = tickets; p.out = ea.out; p.ldo = ea.ldo;
  p.kcache = ea.kcache; p.vcache = ea.vcache; p.row_cache = ea.row_cache; p.row_pos = ea.row_pos;
  p.H = ea.H; p.S_max = ea.S_max; p.D = ea.D; p.kv_fp32 = ea.kv_fp32 ? 1 : 0;
  switch (epi) {
    case G_STORE: LCK(launch_umma_gemm<G_STORE>(s, tA, tA, tB, p, g)); break;
    case G_RESID: LCK(launch_umma_gemm<G_RESID>(s, tA, tA, tB, p, g)); break;
    case G_SWIGLU: LCK(launch_umma_gemm<G_SWIGLU>(s, tA, tA3, tB, p, g)); break;
    default: LCK(launch_umma_gemm<G_QKV>(s, tA, tA, tB, p, g)); break;
  }
  LCK(cudaStreamSynchronize(s));
done:
  return rc;
}

}  // namespace

extern "C" int mvb_linear(const void* d_W, int32_t M, int32_t K, const float* d_x, int32_t ldx, int32_t R,
                          const void* d_gain, float eps, int32_t split_lo, int32_t ksplit_override, float* d_out,
                          int32_t ldo, int32_t accumulate, void* stream) {
  if (!d_W || !d_x || !d_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (K % 64 || R < 1 || R > 128) return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_linear: K %% 64 == 0 and 1 <= R <= 128 required");
  EpiArgs ea{};
  ea.out = d_out; ea.ldo = ldo;
  return run_gemm(accumulate ? G_RESID : G_STORE, d_W, nullptr, M, K, d_x, ldx, R, d_gain, eps, split_lo, ksplit_override, ea,
                  (cudaStream_t)stream);
}

extern "C" int mvb_gemm_test(int32_t epi, const void* d_W, const void* d_W3, int32_t M, int32_t K, const float* d_x, int32_t ldx,
                             int32_t R, const void* d_gain, float eps, int32_t split_lo, int32_t ksplit_override, float* d_out,
                             int32_t ldo, void* d_kcache, void* d_vcache, const int32_t* d_row_cache, const int32_t* d_row_pos,
                             int32_t H, int32_t S_max, int32_t D, int32_t kv_fp32, void* stream) {
  if (!d_W || !d_x || !d_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (epi < G_STORE || epi > G_QKV) return mvb::set_error(MVB_ERR_ARG, "mvb_gemm_test: epilogue %d", epi);
  if (K % 64 || R < 1 || R > 128 || M < 1 || ldo < M || ldx < K)
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_gemm_test: K %% 64 == 0, 1 <= R <= 128, ldo >= M, ldx >= K required");
  if (epi == G_SWIGLU && !d_W3) return mvb::set_error(MVB_ERR_ARG, "mvb_gemm_test: SwiGLU needs W3");
  if (epi == G_QKV) {
    if (!d_kcache || !d_vcache || !d_row_cache || !d_row_pos) return mvb::set_error(MVB_ERR_ARG, "mvb_gemm_test: null KV-cache argument");
    // the scatter splits the K / V thirds of a row into 128-wide heads (head_dim 128, like the stage-1 engine)
    if (D < 128 || D != 128 * H || M != 3 * D || S_max < 1)
      return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_gemm_test: QKV needs D == 128 H, M == 3 D, S_max >= 1");
  }
  EpiArgs ea{};
  ea.out = d_out; ea.ldo = ldo;
  ea.kcache = d_kcache; ea.vcache = d_vcache; ea.row_cache = d_row_cache; ea.row_pos = d_row_pos;
  ea.H = H; ea.S_max = S_max; ea.D = D; ea.kv_fp32 = kv_fp32;
  return run_gemm(epi, d_W, d_W3, M, K, d_x, ldx, R, d_gain, eps, split_lo, ksplit_override, ea, (cudaStream_t)stream);
}
