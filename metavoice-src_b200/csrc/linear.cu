// The weight-streaming tensor-core GEMM: tc_gemm, which the stage-1 and stage-2 engines call, and the standalone
// operator of the C ABI, y[R, M] (+)= f(x)[R, K] . W[M, K]^T with W in bf16, that tests use to check it in isolation.
#include "host.cuh"
#include "tc_gemm.cuh"
#include "tc_gemm_grp.cuh"

using namespace mvb;

namespace mvb {

template <int EPI, int NC, bool SCALED, bool BIASED>
static cudaError_t launch_tc_gemm_nc(cudaStream_t s, const CUtensorMap& tA, const CUtensorMap& tA3, const CUtensorMap& tB,
                                     const GemmP& p, const GemmPlan& g) {
  static PerDeviceOnce attr_set;
  if (attr_set.pending()) {
    cudaError_t e = cudaFuncSetAttribute(k_tc_gemm<EPI, NC, SCALED, BIASED>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_set.mark();
  }
  k_tc_gemm<EPI, NC, SCALED, BIASED><<<dim3(g.tiles, g.ksplit), GEMM_THREADS, g.smem_bytes, s>>>(tA, tA3, tB, p);
  return cudaGetLastError();
}

// The accumulator size is a template parameter (registers): the smallest of 16 / 32 / 64 / 128 columns that holds Rpad.
template <int EPI, bool SCALED, bool BIASED>
static cudaError_t launch_tc_gemm_sc(cudaStream_t s, const CUtensorMap& tA, const CUtensorMap& tA3, const CUtensorMap& tB,
                                     const GemmP& p, const GemmPlan& g) {
  if (p.Rpad <= 16) return launch_tc_gemm_nc<EPI, 2, SCALED, BIASED>(s, tA, tA3, tB, p, g);
  if (p.Rpad <= 32) return launch_tc_gemm_nc<EPI, 4, SCALED, BIASED>(s, tA, tA3, tB, p, g);
  if (p.Rpad <= 64) return launch_tc_gemm_nc<EPI, 8, SCALED, BIASED>(s, tA, tA3, tB, p, g);
  return launch_tc_gemm_nc<EPI, 16, SCALED, BIASED>(s, tA, tA3, tB, p, g);
}

// Instances: int8 row scales on every epilogue but G_GELU, Linear biases on every epilogue, never both (they share
// GemmP's per-row vector slots).
template <int EPI>
static cudaError_t launch_tc_gemm(cudaStream_t s, const CUtensorMap& tA, const CUtensorMap& tA3, const CUtensorMap& tB,
                                  GemmP p, const GemmPlan& g, bool scaled, bool biased) {
  p.ksplit = g.ksplit;
  p.stages = g.stages;
  if constexpr (EPI != G_GELU) {
    if (scaled) return launch_tc_gemm_sc<EPI, true, false>(s, tA, tA3, tB, p, g);
  }
  if (biased) return launch_tc_gemm_sc<EPI, false, true>(s, tA, tA3, tB, p, g);
  if (scaled || biased) return cudaErrorInvalidValue;
  return launch_tc_gemm_sc<EPI, false, false>(s, tA, tA3, tB, p, g);
}

cudaError_t tc_gemm(cudaStream_t s, const TcGemm& a) {
  if (a.Rpad < 16 || a.Rpad > 128 || a.Rpad % 16) return cudaErrorInvalidValue;
  const bool scaled = a.scale != nullptr, biased = a.bias != nullptr;
  if ((a.layer_norm && a.gain == nullptr) || (scaled && biased) || (a.epi == G_SWIGLU && biased && a.bias3 == nullptr))
    return cudaErrorInvalidValue;
  const int NB = a.Rpad * (a.split_lo ? 2 : 1);
  if (a.layer_norm)
    k_prep_b<true><<<a.Rpad, 256, 0, s>>>(a.x, a.ldx, a.gain, a.beta, a.eps, a.K, a.Rpad, a.R, a.split_lo ? 1 : 0, a.B);
  else
    k_prep_b<false><<<a.Rpad, 256, 0, s>>>(a.x, a.ldx, a.gain, nullptr, a.eps, a.K, a.Rpad, a.R, a.split_lo ? 1 : 0, a.B);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  GemmP p{};
  p.M = a.M; p.K = a.K; p.NB = NB; p.Rpad = a.Rpad; p.R = a.R; p.split_lo = a.split_lo ? 1 : 0;
  p.scratch = a.scratch; p.tickets = a.tickets; p.out = a.out; p.ldo = a.ldo;
  p.kcache = a.kcache; p.vcache = a.vcache; p.row_cache = a.row_cache; p.row_pos = a.row_pos;
  p.H = a.H; p.S_max = a.S_max; p.D = a.D; p.kv_fp32 = a.kv_fp32 ? 1 : 0;
  if (scaled) { p.scale = a.scale; p.scale3 = a.scale3; }
  if (biased) { p.bias = a.bias; p.bias3 = a.bias3; }
  const GemmPlan g = plan_gemm(a.M, a.K, NB, a.epi == G_SWIGLU, a.n_sm, a.ksplit);
  const CUtensorMap& tA3 = a.epi == G_SWIGLU ? *a.tmW3 : *a.tmW;
  switch (a.epi) {
    case G_STORE: return launch_tc_gemm<G_STORE>(s, *a.tmW, tA3, *a.tmB, p, g, scaled, biased);
    case G_RESID: return launch_tc_gemm<G_RESID>(s, *a.tmW, tA3, *a.tmB, p, g, scaled, biased);
    case G_SWIGLU: return launch_tc_gemm<G_SWIGLU>(s, *a.tmW, tA3, *a.tmB, p, g, scaled, biased);
    case G_GELU: return launch_tc_gemm<G_GELU>(s, *a.tmW, tA3, *a.tmB, p, g, scaled, biased);
    default: return launch_tc_gemm<G_QKV>(s, *a.tmW, tA3, *a.tmB, p, g, scaled, biased);
  }
}

template <int EPI, int NC, bool BIASED>
static cudaError_t launch_grp_nc(cudaStream_t s, const CUtensorMap& tB, const GemmP& p, const GemmGrp& q, const GemmPlan& g,
                                int units) {
  static PerDeviceOnce attr_set;
  if (attr_set.pending()) {
    cudaError_t e = cudaFuncSetAttribute(k_tc_gemm_grp<EPI, NC, BIASED>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_set.mark();
  }
  k_tc_gemm_grp<EPI, NC, BIASED><<<dim3(g.tiles, p.ksplit, units), GEMM_THREADS, g.smem_bytes, s>>>(tB, p, q);
  return cudaGetLastError();
}

template <int EPI, bool BIASED>
static cudaError_t launch_grp(cudaStream_t s, const CUtensorMap& tB, const GemmP& p, const GemmGrp& q, const GemmPlan& g,
                             int units) {
  if (p.Rpad <= 16) return launch_grp_nc<EPI, 2, BIASED>(s, tB, p, q, g, units);
  if (p.Rpad <= 32) return launch_grp_nc<EPI, 4, BIASED>(s, tB, p, q, g, units);
  if (p.Rpad <= 64) return launch_grp_nc<EPI, 8, BIASED>(s, tB, p, q, g, units);
  return launch_grp_nc<EPI, 16, BIASED>(s, tB, p, q, g, units);
}

template <int EPI>
static cudaError_t launch_grp_b(cudaStream_t s, const CUtensorMap& tB, const GemmP& p, const GemmGrp& q, const GemmPlan& g,
                                int units, bool biased) {
  return biased ? launch_grp<EPI, true>(s, tB, p, q, g, units) : launch_grp<EPI, false>(s, tB, p, q, g, units);
}

cudaError_t tc_gemm_grouped(cudaStream_t s, const TcGemm& a, const TcGemmGrp& g) {
  if (a.Rpad < 16 || a.Rpad > 128 || a.Rpad % 16 || g.n_units < 1 || g.n_units > GEMM_MAX_GROUPS || !g.row_grp || !g.tickets)
    return cudaErrorInvalidValue;
  const bool biased = g.bias[0] != nullptr, normed = g.gain[0] != nullptr;
  if (a.scale != nullptr || (a.layer_norm && !normed)) return cudaErrorInvalidValue;
  const int NB = a.Rpad * (a.split_lo ? 2 : 1);
  PrepGrp pg{};
  pg.row_grp = g.row_grp;
  for (int i = 0; i < GEMM_MAX_GROUPS; ++i) { pg.g2u[i] = g.prep_g2u[i]; pg.gain[i] = g.gain[i]; pg.beta[i] = g.beta[i]; }
  if (a.layer_norm)
    k_prep_b_grp<true><<<a.Rpad, 256, 0, s>>>(a.x, a.ldx, pg, a.eps, a.K, a.Rpad, a.R, a.split_lo ? 1 : 0, a.B);
  else
    k_prep_b_grp<false><<<a.Rpad, 256, 0, s>>>(a.x, a.ldx, pg, a.eps, a.K, a.Rpad, a.R, a.split_lo ? 1 : 0, a.B);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  GemmP p{};
  p.M = a.M; p.K = a.K; p.NB = NB; p.Rpad = a.Rpad; p.R = a.R; p.split_lo = a.split_lo ? 1 : 0;
  p.scratch = a.scratch; p.tickets = g.tickets; p.out = a.out; p.ldo = a.ldo;
  p.kcache = a.kcache; p.vcache = a.vcache; p.row_cache = a.row_cache; p.row_pos = a.row_pos;
  p.H = a.H; p.S_max = a.S_max; p.D = a.D; p.kv_fp32 = a.kv_fp32 ? 1 : 0;
  // K split: the units share the SMs (every split of a tile waits for its siblings, so tiles x splits x units CTAs must
  // be co-resident), and units x splits never exceed the ungrouped launch's splits (its scratch is what is reserved)
  const bool sw = a.epi == G_SWIGLU;
  const GemmPlan full = plan_gemm(a.M, a.K, NB, sw, a.n_sm);
  const int per_unit = a.n_sm / g.n_units > 0 ? a.n_sm / g.n_units : 1;
  const GemmPlan pl = plan_gemm(a.M, a.K, NB, sw, per_unit);
  int ks = pl.ksplit < full.ksplit / g.n_units ? pl.ksplit : full.ksplit / g.n_units;
  if (ks < 1 || pl.tiles > 128) ks = 1;
  p.ksplit = ks;
  p.stages = pl.stages;
  GemmGrp q{};
  q.row_grp = g.row_grp;
  for (int i = 0; i < GEMM_MAX_GROUPS; ++i) {
    q.g2u[i] = g.g2u[i]; q.tmA[i] = g.tmW[i]; q.tmA3[i] = sw ? g.tmW3[i] : g.tmW[i]; q.bias[i] = g.bias[i]; q.bias3[i] = g.bias3[i];
  }
  switch (a.epi) {
    case G_STORE: return launch_grp_b<G_STORE>(s, *a.tmB, p, q, pl, g.n_units, biased);
    case G_RESID: return launch_grp_b<G_RESID>(s, *a.tmB, p, q, pl, g.n_units, biased);
    case G_SWIGLU: return launch_grp_b<G_SWIGLU>(s, *a.tmB, p, q, pl, g.n_units, biased);
    case G_GELU: return launch_grp_b<G_GELU>(s, *a.tmB, p, q, pl, g.n_units, biased);
    default: return launch_grp_b<G_QKV>(s, *a.tmB, p, q, pl, g.n_units, biased);
  }
}

}  // namespace mvb

namespace {

// mvb_linear / mvb_gemm_test: `a` carries the rows, the epilogue and the ksplit override; the B buffer, scratch and
// tickets come from buffers cached per device that only ever grow (no allocation on the steady-state path; this
// standalone operator has no caller-provided workspace, unlike the engine handles).  W3 is the second weight of
// G_SWIGLU.  Synchronises `s`.
int run_gemm(TcGemm a, const void* d_W, const void* d_W3, cudaStream_t s) {
  a.Rpad = (a.R + 15) / 16 * 16;
  const int NB = a.Rpad * (a.split_lo ? 2 : 1);
  int dev = 0;
  if (int e = current_device(&dev, &a.n_sm)) return e;
  const GemmPlan g = plan_gemm(a.M, a.K, NB, a.epi == G_SWIGLU, a.n_sm, a.ksplit);
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
  CUtensorMap tA, tA3, tB;
  MVB_CK(ensure(cB[dev], (size_t)NB * a.K * 2));
  MVB_CK(ensure(cS[dev], sizeof(float) * (g.scratch_floats ? g.scratch_floats : 1)));
  MVB_CK(ensure(cT[dev], sizeof(unsigned) * 256));
  a.B = reinterpret_cast<__nv_bfloat16*>(cB[dev].p);
  a.scratch = reinterpret_cast<float*>(cS[dev].p);
  a.tickets = reinterpret_cast<unsigned*>(cT[dev].p);
  MVB_CK(cudaMemsetAsync(a.B, 0, (size_t)NB * a.K * 2, s));
  MVB_CK(cudaMemsetAsync(a.tickets, 0, sizeof(unsigned) * 256, s));
  if (!make_tmap_bf16(&tA, d_W, (uint64_t)a.M, (uint64_t)a.K, 128) ||
      (a.epi == G_SWIGLU && !make_tmap_bf16(&tA3, d_W3, (uint64_t)a.M, (uint64_t)a.K, 128)) ||
      !make_tmap_bf16(&tB, a.B, (uint64_t)NB, (uint64_t)a.K, (uint32_t)NB))
    return mvb::set_error(MVB_ERR_CUDA, "cuTensorMapEncodeTiled failed");
  a.tmW = &tA; a.tmW3 = &tA3; a.tmB = &tB;
  MVB_CK(tc_gemm(s, a));
  MVB_CK(cudaStreamSynchronize(s));
  return MVB_OK;
}

}  // namespace

namespace mvb {
int tc_gemm_test(const TcGemm& a, const void* d_W, const void* d_W3, void* stream) {
  return run_gemm(a, d_W, d_W3, (cudaStream_t)stream);
}
}  // namespace mvb

extern "C" int mvb_linear(const void* d_W, int32_t M, int32_t K, const float* d_x, int32_t ldx, int32_t R,
                          const void* d_gain, float eps, int32_t split_lo, int32_t ksplit_override, float* d_out,
                          int32_t ldo, int32_t accumulate, void* stream) {
  if (!d_W || !d_x || !d_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (K % 64 || R < 1 || R > 128) return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_linear: K %% 64 == 0 and 1 <= R <= 128 required");
  TcGemm a{};
  a.epi = accumulate ? G_RESID : G_STORE;
  a.x = d_x; a.ldx = ldx; a.gain = reinterpret_cast<const __nv_bfloat16*>(d_gain); a.eps = eps;
  a.M = M; a.K = K; a.R = R; a.split_lo = split_lo; a.ksplit = ksplit_override;
  a.out = d_out; a.ldo = ldo;
  return run_gemm(a, d_W, nullptr, (cudaStream_t)stream);
}

namespace {

int gemm_test(int32_t epi, const void* d_W, const void* d_W3, const void* d_scale, const void* d_scale3, int32_t M, int32_t K,
              const float* d_x, int32_t ldx, int32_t R, const void* d_gain, float eps, int32_t split_lo, int32_t ksplit_override,
              float* d_out, int32_t ldo, void* d_kcache, void* d_vcache, const int32_t* d_row_cache, const int32_t* d_row_pos,
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
  TcGemm a{};
  a.epi = epi;
  a.x = d_x; a.ldx = ldx; a.gain = reinterpret_cast<const __nv_bfloat16*>(d_gain); a.eps = eps;
  a.M = M; a.K = K; a.R = R; a.split_lo = split_lo; a.ksplit = ksplit_override;
  a.out = d_out; a.ldo = ldo;
  a.kcache = d_kcache; a.vcache = d_vcache; a.row_cache = d_row_cache; a.row_pos = d_row_pos;
  a.H = H; a.S_max = S_max; a.D = D; a.kv_fp32 = kv_fp32;
  a.scale = reinterpret_cast<const __nv_bfloat16*>(d_scale); a.scale3 = reinterpret_cast<const __nv_bfloat16*>(d_scale3);
  return run_gemm(a, d_W, d_W3, (cudaStream_t)stream);
}

}  // namespace

extern "C" int mvb_gemm_test(int32_t epi, const void* d_W, const void* d_W3, int32_t M, int32_t K, const float* d_x, int32_t ldx,
                             int32_t R, const void* d_gain, float eps, int32_t split_lo, int32_t ksplit_override, float* d_out,
                             int32_t ldo, void* d_kcache, void* d_vcache, const int32_t* d_row_cache, const int32_t* d_row_pos,
                             int32_t H, int32_t S_max, int32_t D, int32_t kv_fp32, void* stream) {
  return gemm_test(epi, d_W, d_W3, nullptr, nullptr, M, K, d_x, ldx, R, d_gain, eps, split_lo, ksplit_override, d_out, ldo,
                   d_kcache, d_vcache, d_row_cache, d_row_pos, H, S_max, D, kv_fp32, stream);
}

extern "C" int mvb_w8_gemm_test(int32_t epi, const void* d_W, const void* d_W3, const void* d_scale, const void* d_scale3,
                                int32_t M, int32_t K, const float* d_x, int32_t ldx, int32_t R, const void* d_gain, float eps,
                                int32_t split_lo, int32_t ksplit_override, float* d_out, int32_t ldo, void* d_kcache,
                                void* d_vcache, const int32_t* d_row_cache, const int32_t* d_row_pos, int32_t H, int32_t S_max,
                                int32_t D, int32_t kv_fp32, void* stream) {
  if (!d_scale || (epi == G_SWIGLU && !d_scale3)) return mvb::set_error(MVB_ERR_ARG, "mvb_w8_gemm_test: null row scales");
  return gemm_test(epi, d_W, d_W3, d_scale, d_scale3, M, K, d_x, ldx, R, d_gain, eps, split_lo, ksplit_override, d_out, ldo,
                   d_kcache, d_vcache, d_row_cache, d_row_pos, H, S_max, D, kv_fp32, stream);
}

extern "C" int mvb_s2_linear_test(int32_t epi, int32_t norm, const void* d_W, const void* d_W3, const void* d_bias,
                                  const void* d_bias3, int32_t M, int32_t K, const float* d_x, int32_t ldx, int32_t R,
                                  const void* d_gain, const void* d_beta, float eps, int32_t split_lo, int32_t ksplit_override,
                                  float* d_out, int32_t ldo, void* stream) {
  if (!d_W || !d_x || !d_out) return mvb::set_error(MVB_ERR_ARG, "null argument");
  if (epi != G_STORE && epi != G_RESID && epi != G_SWIGLU && epi != G_GELU)
    return mvb::set_error(MVB_ERR_ARG, "mvb_s2_linear_test: epilogue %d", epi);
  if (norm < 0 || norm > 2) return mvb::set_error(MVB_ERR_ARG, "mvb_s2_linear_test: norm %d", norm);
  if ((norm != 0) != (d_gain != nullptr) || (d_beta && norm != 2))
    return mvb::set_error(MVB_ERR_ARG, "mvb_s2_linear_test: a norm takes a gain (and only LayerNorm a beta)");
  if (K % 64 || R < 1 || R > 128 || M < 1 || ldo < M || ldx < K)
    return mvb::set_error(MVB_ERR_UNSUPPORTED, "mvb_s2_linear_test: K %% 64 == 0, 1 <= R <= 128, ldo >= M, ldx >= K required");
  if (epi == G_SWIGLU && (!d_W3 || (d_bias && !d_bias3)))
    return mvb::set_error(MVB_ERR_ARG, "mvb_s2_linear_test: SwiGLU needs W3 (and bias3 with a bias)");
  TcGemm a{};
  a.epi = epi;
  a.x = d_x; a.ldx = ldx; a.gain = reinterpret_cast<const __nv_bfloat16*>(d_gain); a.eps = eps;
  a.layer_norm = norm == 2; a.beta = reinterpret_cast<const __nv_bfloat16*>(d_beta);
  a.M = M; a.K = K; a.R = R; a.split_lo = split_lo; a.ksplit = ksplit_override;
  a.out = d_out; a.ldo = ldo;
  a.bias = reinterpret_cast<const __nv_bfloat16*>(d_bias);
  a.bias3 = epi == G_SWIGLU ? reinterpret_cast<const __nv_bfloat16*>(d_bias3) : nullptr;
  return run_gemm(a, d_W, d_W3, (cudaStream_t)stream);
}
