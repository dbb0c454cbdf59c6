// Host-side helpers for the tensor-core GEMM path: TMA tensor maps (driver entry point resolved at run
// time, so libmvb200 does not link libcuda) and launch configuration.
#pragma once
#include <cuda.h>
#include <stdlib.h>
#include <cuda_runtime.h>

#include "umma_gemm.cuh"

namespace mvb {

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

// Pick the K split so that (row tiles x splits) fills the SMs about once, and the deepest ring that fits.
static inline GemmPlan plan_gemm(int M, int K, int NB, bool swiglu, int n_sm) {
  GemmPlan g;
  g.tiles = (M + 127) / 128;
  const int nkb = K / 64;
  int ks = n_sm / g.tiles;
  if (ks < 1) ks = 1;
  if (ks > nkb / 2) ks = nkb / 2 > 0 ? nkb / 2 : 1;   // at least two k-blocks per split: tiny K is latency-, not bandwidth-bound
  if (nkb <= 8 && getenv("MVB_GEMM_SPLIT_TINY") == nullptr) ks = 1;   // K <= 512 (stage-2 width): the split-K hand-off costs more than it buys
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
  g.scratch_floats = (size_t)g.tiles * ks * (swiglu ? 2 : 1) * NB * 128;
  return g;
}

template <int EPI, int NC>
static inline cudaError_t launch_umma_gemm_nc(cudaStream_t s, const CUtensorMap& tA, const CUtensorMap& tA3, const CUtensorMap& tB,
                                              const GemmP& p, const GemmPlan& g) {
  static PerDeviceOnce attr_set;
  if (attr_set.pending()) {
    cudaError_t e = cudaFuncSetAttribute(k_umma_gemm<EPI, NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_set.mark();
  }
  k_umma_gemm<EPI, NC><<<dim3(g.tiles, g.ksplit), GEMM_THREADS, g.smem_bytes, s>>>(tA, tA3, tB, p);
  return cudaGetLastError();
}

// The accumulator size is a template parameter (registers): the smallest of 16 / 32 / 64 / 128 columns that holds Rpad.
template <int EPI>
static inline cudaError_t launch_umma_gemm(cudaStream_t s, const CUtensorMap& tA, const CUtensorMap& tA3, const CUtensorMap& tB,
                                           GemmP p, const GemmPlan& g) {
  if (p.Rpad < 16 || p.Rpad > 128 || p.Rpad % 16) return cudaErrorInvalidValue;
  p.ksplit = g.ksplit;
  p.stages = g.stages;
  if (p.Rpad <= 16) return launch_umma_gemm_nc<EPI, 2>(s, tA, tA3, tB, p, g);
  if (p.Rpad <= 32) return launch_umma_gemm_nc<EPI, 4>(s, tA, tA3, tB, p, g);
  if (p.Rpad <= 64) return launch_umma_gemm_nc<EPI, 8>(s, tA, tA3, tB, p, g);
  return launch_umma_gemm_nc<EPI, 16>(s, tA, tA3, tB, p, g);
}

}  // namespace mvb
