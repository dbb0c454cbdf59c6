// sm_90a building blocks of the tensor-core kernels: mbarrier ring, TMA (cp.async.bulk.tensor) and bulk copies into
// 128B-swizzled shared memory, ldmatrix + mma.sync fragment loads, the two-term bf16 activation split, and the TMA ->
// mma.sync mainloop shared by the weight-streaming GEMM and the MBD convolution.
// Hand-written inline PTX (fragment layouts: PTX ISA, ldmatrix and mma.m16n8k16).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace mvb {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) trap_if_stuck(t0);
}

// ---- TMA and bulk copies ----------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tensormap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// Tile loads: c0 = element offset along the contiguous (K) dimension, c1 = row offset, c2 = outer index.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_hint(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_3d_hint(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "l"(policy) : "memory");
}
// Contiguous global -> shared copy (no tensor map), completing on `bar`.
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// Generic-proxy shared-memory writes -> visible to the async proxy (TMA, and the operands the tensor core reads).
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

}  // namespace ptx

// Bytes from the start of the dynamic shared memory to its first 1024-byte aligned byte (the 128B-swizzled tiles need
// it).  Use as `smem_raw + smem_pad_1024(smem_raw)`: pointer arithmetic on the shared array itself.  An integer round
// trip would lose the .shared state space and turn every access into a generic LD/ST; even an inlined helper that
// returns the pointer changes the decode kernel's register allocation.
__device__ __forceinline__ uint32_t smem_pad_1024(const void* smem_raw) {
  return (1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u;
}

// Slot and mbarrier parity of use number `it` of a ring of S slots.
struct RingPos {
  uint32_t stage, phase;
};
__device__ __forceinline__ RingPos ring_pos(uint32_t it, uint32_t S) { return {it % S, (it / S) & 1u}; }

// ---- ldmatrix + mma.sync ----------------------------------------------------------------------
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

// D[16x8] += A[16x16] * B[16x8], bf16 operands, fp32 accumulate (fragment layouts: PTX ISA, mma.m16n8k16)
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// byte offset of 16-byte chunk `ch` of row `row` in a K-major tile of 128-byte rows written with the 128B swizzle
// (TMA CU_TENSOR_MAP_SWIZZLE_128B; the tile base is 1024-byte aligned)
__device__ __forceinline__ uint32_t sw128_off(int row, int ch) { return (uint32_t)(row * 128 + ((ch ^ (row & 7)) << 4)); }

// Fragments of k-step kk (k = 16 kk .. 16 kk + 15) from a K-major 128B-swizzled tile of 64 bf16 per row; q = lane / 8
// and r8 = lane % 8 pick the row and 16-byte chunk whose address this lane supplies to ldmatrix.x4.
// A operand: rows row0 .. row0 + 15.
__device__ __forceinline__ void ldsm_a(uint32_t tile, int row0, int kk, int q, int r8, uint32_t (&a)[4]) {
  ldsm_x4(tile + sw128_off(row0 + r8 + ((q & 1) << 3), 2 * kk + (q >> 1)), a);
}
// B operands of two n8 chunks: rows row0 .. row0 + 7 in b[0], b[1] and rows row0 + 8 .. row0 + 15 in b[2], b[3].
__device__ __forceinline__ void ldsm_b(uint32_t tile, int row0, int kk, int q, int r8, uint32_t (&b)[4]) {
  ldsm_x4(tile + sw128_off(row0 + r8 + ((q >> 1) << 3), 2 * kk + (q & 1)), b);
}

// Exact two-term bf16 split of an activation, x = hi + lo to 2^-17 (16 mantissa bits): hi = bf16(x), lo = lo_term(x, hi).
__device__ __forceinline__ __nv_bfloat16 lo_term(float x, __nv_bfloat16 hi) { return __float2bfloat16_rn(x - __bfloat162float(hi)); }
// (x0, x1) -> packed bf16 pair of the high terms and of the low terms
__device__ __forceinline__ void pack_hi_lo(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat16 h0 = __float2bfloat16_rn(x0), h1 = __float2bfloat16_rn(x1);
  const __nv_bfloat16 l0 = lo_term(x0, h0), l1 = lo_term(x1, h1);
  hi = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
  lo = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
}

// ---- TMA -> mma.sync mainloop (288 threads) ---------------------------------------------------
// An S-stage ring of stage_bytes each at `smem`, its full[S] / empty[S] mbarriers right behind it.
//   * warp 0 = producer: for iteration `it` it waits until the stage is drained, arms the full barrier with stage_bytes
//     and lets one elected lane call issue(it, stage smem address, full barrier) to start the stage's TMA loads.
//   * warps 1..8 = consumers: warp w multiplies weight rows [16 (w - 1), 16 w) of the NA A tiles (128 rows x 64 k
//     each, at the stage base) by the first nc n8 chunks of the B tile at stage + b_off, and (split_lo) by the lo rows
//     that start lo_row rows further, into the same fp32 accumulator acc[a][chunk].
// Returns false in the producer warp and true in the consumer warps, which then own acc.
template <int NA, int NC, typename Issue>
__device__ __forceinline__ bool tc_mainloop(uint8_t* smem, uint32_t S, uint32_t stage_bytes, uint32_t b_off, int n_it, int nc,
                                            int lo_row, bool split_lo, const Issue& issue, float (&acc)[NA][NC][4]) {
  constexpr uint32_t A_BYTES = 128 * 64 * 2;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)S * stage_bytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (uint32_t s = 0; s < S; ++s) {
      ptx::mbar_init(ptx::smem_u32(bars + s), 1);
      ptx::mbar_init(ptx::smem_u32(bars + S + s), 8);   // one arrive per consumer warp
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // the whole warp walks the loop (uniform operands), one elected lane issues
    for (int it = 0; it < n_it; ++it) {
      const RingPos rp = ring_pos(it, S);
      ptx::mbar_wait(ptx::smem_u32(bars + S + rp.stage), rp.phase ^ 1u);
      if (ptx::elect_one()) {
        const uint32_t full = ptx::smem_u32(bars + rp.stage);
        ptx::mbar_arrive_expect_tx(full, stage_bytes);
        issue(it, ptx::smem_u32(smem + (size_t)rp.stage * stage_bytes), full);
      }
      __syncwarp();
    }
    return false;
  }

  const int w16 = 16 * (warp - 1);
#pragma unroll
  for (int a = 0; a < NA; ++a)
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[a][c][e] = 0.f;
  for (int it = 0; it < n_it; ++it) {
    const RingPos rp = ring_pos(it, S);
    ptx::mbar_wait(ptx::smem_u32(bars + rp.stage), rp.phase);
    const uint32_t st = ptx::smem_u32(smem + (size_t)rp.stage * stage_bytes);
    const uint32_t bst = st + b_off;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t af[NA][4];
#pragma unroll
      for (int a = 0; a < NA; ++a) ldsm_a(st + a * A_BYTES, w16, kk, lane >> 3, lane & 7, af[a]);
#pragma unroll
      for (int g = 0; g < NC / 2; ++g) {
        if (2 * g >= nc) break;
#pragma unroll
        for (int half = 0; half < 2; ++half) {   // hi rows, then (split_lo) the lo rows into the same accumulator
          if (half == 1 && !split_lo) break;
          uint32_t b[4];
          ldsm_b(bst, half * lo_row + 16 * g, kk, lane >> 3, lane & 7, b);
#pragma unroll
          for (int a = 0; a < NA; ++a) {
            mma_bf16_16816(acc[a][2 * g], af[a], b[0], b[1]);
            mma_bf16_16816(acc[a][2 * g + 1], af[a], b[2], b[3]);
          }
        }
      }
    }
    __syncwarp();                          // every lane's fragment loads of this stage are done
    if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(bars + S + rp.stage));
  }
  return true;
}

}  // namespace mvb
