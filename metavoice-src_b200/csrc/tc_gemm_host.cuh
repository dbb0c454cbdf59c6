// Host side of the tensor-core kernels: TMA tensor maps (driver entry point resolved at run time, so libmvb200 does
// not link libcuda), the weight-streaming GEMM's launch plan, and its one entry point tc_gemm (linear.cu).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace mvb {

enum { G_STORE = 0, G_RESID = 1, G_SWIGLU = 2, G_QKV = 3, G_GELU = 4 };

constexpr int GEMM_A_BYTES = 128 * 64 * 2;  // one 128-row x 64-k bf16 tile
// SM count the engine workspaces size the split-K scratch for.  plan_gemm never plans for more SMs, so the reserved
// scratch always covers the plan of a launch (132: H100 SXM, the largest sm_90 part).
constexpr int GEMM_MAX_SM = 132;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// bf16 row-major [rows, cols] -> tiles of [box_rows, 64] with the 128-byte swizzle the MMA fragment loads expect.
static inline bool make_tmap_bf16(CUtensorMap* tm, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// 3-D tensor map over one matrix kind of every layer: dims {K, M, n_layer}, tile {64, 128, 1}, 128B swizzle.
static inline bool make_tmap_bf16_3d(CUtensorMap* tm, const void* ptr, uint64_t K, uint64_t M, uint64_t L, uint64_t layer_stride_bytes,
                              uint32_t tile_rows) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return false;
  cuuint64_t dims[3] = {K, M, L};
  cuuint64_t strides[2] = {K * 2, layer_stride_bytes};
  cuuint32_t box[3] = {64u, tile_rows, 1};              // rows past M read as zero
  cuuint32_t estr[3] = {1, 1, 1};
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct GemmPlan {
  int ksplit, stages;
  size_t smem_bytes, scratch_floats;
  int tiles;
};

// Pick the K split so that (row tiles x splits) fills the SMs (at most GEMM_MAX_SM) about once, and the deepest ring
// that fits.
// ksplit_override > 0 forces the split instead, capped so that every split of a tile stays co-resident.
static inline GemmPlan plan_gemm(int M, int K, int NB, bool swiglu, int n_sm, int ksplit_override = 0) {
  GemmPlan g;
  if (n_sm > GEMM_MAX_SM) n_sm = GEMM_MAX_SM;
  g.tiles = (M + 127) / 128;
  const int nkb = K / 64;
  int ks = n_sm / g.tiles;
  if (ks < 1) ks = 1;
  if (ks > nkb / 2) ks = nkb / 2 > 0 ? nkb / 2 : 1;   // at least two k-blocks per split: tiny K is latency-, not bandwidth-bound
  if (nkb <= 8) ks = 1;                                // K <= 512 (stage-2 width): the split-K hand-off costs more than it buys
  if (ks > 16) ks = 16;
  if (g.tiles > 128) ks = 1;                           // (the split-K arrival counters cover 128 tiles)
  g.ksplit = ks;
  const int stage_bytes = (swiglu ? 2 : 1) * GEMM_A_BYTES + NB * 128;
  int st = (200 * 1024) / stage_bytes;
  if (st > 8) st = 8;
  if (st < 2) st = 2;
  const int per = (nkb + ks - 1) / ks;
  if (st > per) st = per < 2 ? 2 : per;
  g.stages = st;
  g.smem_bytes = 1024 + (size_t)st * stage_bytes + 2 * st * 8 + 64;
  if (ksplit_override > 0) {
    // every split of a tile waits for its siblings inside the kernel: all tiles x ksplit CTAs must be co-resident
    const int cap = n_sm / g.tiles > 0 ? n_sm / g.tiles : 1;
    g.ksplit = ksplit_override < cap ? ksplit_override : cap;
    if (g.tiles > 128) g.ksplit = 1;
  }
  g.scratch_floats = (size_t)g.tiles * g.ksplit * (swiglu ? 2 : 1) * NB * 128;
  return g;
}

// One projection on the tensor cores: k_prep_b stages the R input rows (optional RMSNorm or LayerNorm, then the bf16
// hi / lo split) in B, then k_tc_gemm computes out[n, j] (+)= f(x)[n, :] . W[j, :] (+ bias[j]) with epilogue `epi`.
struct TcGemm {
  int epi;                                        // G_STORE / G_RESID / G_SWIGLU / G_QKV / G_GELU
  const CUtensorMap* tmW;                         // weight [M, K], 128-row boxes
  const CUtensorMap* tmW3;                        // G_SWIGLU: the second weight (silu(x W^T) * (x W3^T))
  __nv_bfloat16* B;                               // activation operand [Rpad * (1 + split_lo), K]
  const CUtensorMap* tmB;                         // map over B with one box of all its rows
  const float* x; int ldx;                        // input rows
  const __nv_bfloat16* gain; float eps;           // RMSNorm (LayerNorm when layer_norm) gain, or null: no norm
  int layer_norm;                                 // with gain: LayerNorm, (x - mean) * rstd * gain (+ beta)
  const __nv_bfloat16* beta;                      // LayerNorm bias, or null
  int M, K;
  int R, Rpad, split_lo;                          // rows, rows reserved in B (multiple of 16, <= 128), lo terms carried
  float* out; int ldo;
  void* kcache; void* vcache;                     // G_QKV: KV-cache scatter of the k / v thirds
  const int* row_cache; const int* row_pos;
  int H, S_max, D, kv_fp32;
  float* scratch;                                 // split-K partial tiles: plan_gemm(...).scratch_floats
  unsigned* tickets;                              // [256] split-K counters, zero before the first launch
  int n_sm;                                       // SMs of the device
  int ksplit;                                     // > 0: force the K split (tests)
  const __nv_bfloat16* scale;                     // int8 weights: bf16 [M] row scales of W, or null
  const __nv_bfloat16* scale3;                    // G_SWIGLU: those of W3
  const __nv_bfloat16* bias;                      // bf16 [M] Linear bias of W, or null (never with scale)
  const __nv_bfloat16* bias3;                     // G_SWIGLU with bias: that of W3
};
cudaError_t tc_gemm(cudaStream_t s, const TcGemm& a);

// tc_gemm grouped over up to GEMM_MAX_GROUPS units with their own weights (tc_gemm_grp.cuh): `a` gives what every unit
// shares (rows, epilogue, output, cache, B buffer and its map, scratch, SM count; a.tmW / a.gain / a.beta / a.bias are
// unused), `g` each row's voice group and, per voice group, its unit of the norm prologue and of the GEMM.  One
// k_prep_b_grp and one k_tc_gemm_grp launch; the K split is chosen so that tiles x splits x units fit the SMs once and
// the split-K scratch stays within what a.scratch holds for one ungrouped launch of the same shape.
constexpr int GEMM_MAX_GROUPS = 16;
struct TcGemmGrp {
  const int* row_grp;                                  // [R] voice group of each activation row (device)
  unsigned* tickets;                                   // [GEMM_MAX_GROUPS * 256] split-K counters, zero before first use
  int n_units;                                         // GEMM units (distinct weights)
  int g2u[GEMM_MAX_GROUPS];                            // voice group -> GEMM unit
  const CUtensorMap* tmW[GEMM_MAX_GROUPS];             // per GEMM unit, maps in DEVICE memory
  const CUtensorMap* tmW3[GEMM_MAX_GROUPS];
  const __nv_bfloat16* bias[GEMM_MAX_GROUPS];          // per GEMM unit (all null, or all set)
  const __nv_bfloat16* bias3[GEMM_MAX_GROUPS];
  int prep_g2u[GEMM_MAX_GROUPS];                       // voice group -> norm unit
  const __nv_bfloat16* gain[GEMM_MAX_GROUPS];          // per norm unit (all null: no norm)
  const __nv_bfloat16* beta[GEMM_MAX_GROUPS];
};
cudaError_t tc_gemm_grouped(cudaStream_t s, const TcGemm& a, const TcGemmGrp& g);
// Test hooks: tc_gemm over `a` with the B buffer, split-K scratch and tickets of mvb_linear (a.Rpad, a.B, a.scratch,
// a.tickets, a.n_sm and the tensor maps are filled in); W3 is G_SWIGLU's second weight.  Synchronises `stream`.
int tc_gemm_test(const TcGemm& a, const void* d_W, const void* d_W3, void* stream);

}  // namespace mvb
