// Shared device helpers for libmvb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#define MVB_WARP 32

namespace mvb {

// cudaFuncSetAttribute applies to the CURRENT device only: remember per (call site, device), not per process.
struct PerDeviceOnce {
  bool done[64] = {};
  bool pending() const { int d = 0; cudaGetDevice(&d); return d < 0 || d >= 64 || !done[d]; }
  void mark() { int d = 0; cudaGetDevice(&d); if (d >= 0 && d < 64) done[d] = true; }
};

// 128-bit streaming load that does not pollute L1 (weights/KV are read exactly once per step).
__device__ __forceinline__ uint4 ldg_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// bf16 pair packed in a 32-bit word -> two fp32 (exact).
__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

__device__ __forceinline__ float bf16_to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// acc += dot(8 bf16 weights in w, 8 fp32 activations in (a, b))
__device__ __forceinline__ void fma8(float& acc, const uint4& w, const float4& a, const float4& b) {
  acc = fmaf(bf_lo(w.x), a.x, acc);
  acc = fmaf(bf_hi(w.x), a.y, acc);
  acc = fmaf(bf_lo(w.y), a.z, acc);
  acc = fmaf(bf_hi(w.y), a.w, acc);
  acc = fmaf(bf_lo(w.z), b.x, acc);
  acc = fmaf(bf_hi(w.z), b.y, acc);
  acc = fmaf(bf_lo(w.w), b.z, acc);
  acc = fmaf(bf_hi(w.w), b.w, acc);
}

// Bound of every spin wait (mbarrier, grid counter): 4e9 cycles (~2 s at H100 clocks).  A protocol bug must surface as
// a launch failure, never as a hung GPU.
__device__ __forceinline__ void trap_if_stuck(long long t0) {
  if (clock64() - t0 > 4000000000ll) __trap();
}

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_inc(unsigned* p) {
  asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p) : "memory");
}
// Grid-wide counter wait: spin until *ctr >= target, with acquire ordering (pairs with red_release_inc / atomics).
__device__ __forceinline__ void wait_counter(const unsigned* ctr, unsigned target) {
  const long long t0 = clock64();
  while (ld_acquire_u32(ctr) < target) trap_if_stuck(t0);
}

// Programmatic dependent launch: let the next kernel in the stream start its independent
// prologue early / wait for the previous kernel's memory to be visible.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Philox4x32-10 counter-based RNG (Salmon et al. 2011), used for the on-device Exp(1) noise.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}

// Exp(1) draw from one Philox word: uni = ((x >> 8) + 0.5) 2^-24 lies in (0, 1) in real arithmetic, but in fp32 the
// top value 2^24 - 0.5 rounds to 2^24, i.e. uni = 1 and q = -0, and a score p / q of -inf (p > 0) or NaN (p = 0, a
// dropped entry) wins the unsigned arg-max.  That value is clamped to the largest float below 1; every other draw is
// unchanged.
__device__ __forceinline__ float philox_exp1(uint32_t x) {
  const float uni = fminf(((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f), 0x1.fffffep-1f);
  return -logf(uni);
}

}  // namespace mvb
