// Weight-only int4 stage-1 kernels (quantisation_mode="int4", fast_inference_utils.py:297-306): the int4 counterpart of
// k_gemv for decode (path A) and the per-layer dequantiser that feeds the bf16 tensor-core GEMM for prefill (path B).
//
// Packed matrix [M, K] (K % 256 == 0; layout in include/mvb200.h, produced only by mvb200/quantize.py:pack_matrix):
//   nibbles  uint32 [M][K/8]: word w of row m holds q(8w + 2i) in bits 4i..4i+3 and q(8w + 2i + 1) in bits 16+4i..19+4i
//            (i = 0..3), so one shift and one mask put the pair (2i, 2i + 1) into the two bf16 halves of a register;
//   then, at the next 256-byte boundary, bf16 [M][K/128][2] = {scale s, zero z} of each 128-wide group of a row.
// Dequantised weight (both kernels, bit for bit): W_deq = bf16_rn((q - 8) s + z), the exact value rounded once
// (fma.rn.bf16x2).
#pragma once
#include "stage1_kernels.cuh"

namespace mvb {

constexpr int W4_GROUP = 128;

__host__ __device__ inline size_t w4_sz_offset(int M, int K) { return ((size_t)M * K / 2 + 255) / 256 * 256; }
__host__ __device__ inline size_t w4_packed_bytes(int M, int K) { return w4_sz_offset(M, K) + (size_t)M * (K / W4_GROUP) * 4; }

// Pair i (k = 8w + 2i, 8w + 2i + 1) of a packed word -> their two W_deq values as one bf16x2 word (low half = the lower
// k).  0x4300 | q is the bf16 128 + q (exact: the bf16 ulp at 128 is 1), so subtracting 136 gives q - 8 exactly; the
// bf16x2 fma then rounds (q - 8) s + z once.  sz2 = {s, s}, zz2 = {z, z}.
__device__ __forceinline__ uint32_t w4_deq_pair(uint32_t w, int i, __nv_bfloat162 s2, __nv_bfloat162 z2) {
  const uint32_t v = ((w >> (4 * i)) & 0x000F000Fu) | 0x43004300u;
  const __nv_bfloat162 q = __hsub2(*reinterpret_cast<const __nv_bfloat162*>(&v), __float2bfloat162_rn(136.f));
  const __nv_bfloat162 r = __hfma2(q, s2, z2);
  return *reinterpret_cast<const uint32_t*>(&r);
}

// Position of activation k in k_gemv_w4's shared-memory layout.  In a tile of W = min(512, K - tb) values starting at
// tb = k & ~511, lane j of a half-warp owns k in [tb + 32 j, tb + 32 j + 32); its i-th float4 of them sits at
// tb + i (W / 8) + 4 j, so the 16 lanes of a half-warp read 16 consecutive float4 per step (no bank conflicts; the two
// half-warps work on different tiles).
__device__ __forceinline__ int w4_perm(int k, int K) {
  const int tb = k & ~511;
  const int W = (K - tb) < 512 ? (K - tb) : 512;
  const int r = k - tb, j = r >> 5, i = r & 31;
  return tb + (i >> 2) * (W >> 3) + (j << 2) + (i & 3);
}

// 32 consecutive k of two weight rows (va, vb: one 128-bit load each, scale / zero in sa, sb) against the two CFG
// activation rows (x0, x1: float4 i of the lane at x[i * xstride]).  Sequential fp32 fmas in k order.
__device__ __forceinline__ void w4_dot32(const uint4& va, __nv_bfloat162 sza, const uint4& vb, __nv_bfloat162 szb, const float4* x0,
                                         const float4* x1, int xstride, float& a00, float& a01, float& a10, float& a11) {
  const uint32_t wa[4] = {va.x, va.y, va.z, va.w}, wb[4] = {vb.x, vb.y, vb.z, vb.w};
  const __nv_bfloat162 sa2 = __low2bfloat162(sza), za2 = __high2bfloat162(sza);
  const __nv_bfloat162 sb2 = __low2bfloat162(szb), zb2 = __high2bfloat162(szb);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float4 p = x0[(2 * c + h) * xstride], q = x1[(2 * c + h) * xstride];
      const float xp[4] = {p.x, p.y, p.z, p.w}, xq[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const uint32_t da = w4_deq_pair(wa[c], 2 * h + e, sa2, za2);
        const uint32_t db = w4_deq_pair(wb[c], 2 * h + e, sb2, zb2);
        const float wa0 = bf_lo(da), wa1 = bf_hi(da), wb0 = bf_lo(db), wb1 = bf_hi(db);
        a00 = fmaf(wa0, xp[2 * e], a00); a00 = fmaf(wa1, xp[2 * e + 1], a00);
        a01 = fmaf(wa0, xq[2 * e], a01); a01 = fmaf(wa1, xq[2 * e + 1], a01);
        a10 = fmaf(wb0, xp[2 * e], a10); a10 = fmaf(wb1, xp[2 * e + 1], a10);
        a11 = fmaf(wb0, xq[2 * e], a11); a11 = fmaf(wb1, xq[2 * e + 1], a11);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// k_gemv's contract (GemvP, the RMSNorm prologue, the four epilogues, gridDim.y = utterances) over int4 packed weights:
// p.W (and p.W3 for EPI_SWIGLU) point at packed matrices.  A warp owns one item, as in k_gemv (rows 2i, 2i + 1, or w1 row
// i and w3 row i).  K is cut into NT = ceil(K / 512) tiles of 512 (a trailing one of 256 when K % 512 == 256) dealt
// alternately to the two half-warps; lane j of a half-warp streams 32 nibbles of each row per tile with one 128-bit load
// per row, reads that group's (scale, zero) once, and prefetches its next tile while it consumes the current one (lanes
// 0-7 take the trailing 256-wide tile).  Per output a lane's fp32 sum runs over at most 32 ceil(NT / 2) products in k
// order, then a 5-level butterfly adds the 32 lanes.
// Memory pipeline: the weights do not depend on the previous kernel, so before griddepcontrol.wait every warp asks L2 for
// all the rows (and their scale / zero pairs) it will stream, one bulk prefetch per item and lane: the whole matrix is in
// flight while the previous kernel drains and the activations are staged, and the main loop then reads L2.
// The prologue and the epilogues are k_gemv's (gemv_prologue / gemv_epilogue, stage1_kernels.cuh) over the w4_perm layout.
template <int EPI>
__global__ void __launch_bounds__(256, 2) k_gemv_w4(GemvP p, S1State st) {
  extern __shared__ float xs[];  // [2][K] in the w4_perm layout
  __shared__ float red[16];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, half = lane >> 4, j = lane & 15;
  const int K = p.K;
  const int n_items = (EPI == EPI_SWIGLU) ? p.M : (p.M >> 1);
  const int G = K / W4_GROUP;
  const size_t rowb = (size_t)K >> 1;
  const uint8_t* Wn = reinterpret_cast<const uint8_t*>(p.W);
  const __nv_bfloat162* Wsz = reinterpret_cast<const __nv_bfloat162*>(Wn + w4_sz_offset(p.M, K));
  const uint8_t* W3n = reinterpret_cast<const uint8_t*>(p.W3);
  const __nv_bfloat162* W3sz = EPI == EPI_SWIGLU ? reinterpret_cast<const __nv_bfloat162*>(W3n + w4_sz_offset(p.M, K)) : nullptr;
  pdl_launch_dependents();
  {
    // lane n of a warp prefetches the warp's n-th item (the loop below visits the same items in the same order)
    const int item = blockIdx.x * 8 + warp + lane * gridDim.x * 8;
    if (item < n_items) {
      if (EPI == EPI_SWIGLU) {
        l2_prefetch(Wn + (size_t)item * rowb, rowb);
        l2_prefetch(W3n + (size_t)item * rowb, rowb);
        l2_prefetch(Wsz + (size_t)item * G, (size_t)G * 4);
        l2_prefetch(W3sz + (size_t)item * G, (size_t)G * 4);
      } else {
        l2_prefetch(Wn + (size_t)(2 * item) * rowb, 2 * rowb);
        l2_prefetch(Wsz + (size_t)(2 * item) * G, (size_t)G * 8);
      }
    }
  }
  pdl_wait();  // activations written by the previous kernel are now visible

  const int u = st.slot_map[blockIdx.y];
  gemv_prologue(p, 2 * u, xs, red, [K](int k) { return w4_perm(k, K); });

  const int KF = K >> 9;               // full 512-wide tiles
  const bool tail = (K & 511) != 0;    // one trailing 256-wide tile

  const int NT = KF + (tail ? 1 : 0);   // tiles; tile t belongs to half-warp t & 1
  for (int item = blockIdx.x * 8 + warp; item < n_items; item += gridDim.x * 8) {
    const uint8_t *na, *nb;
    const __nv_bfloat162 *sa, *sb;
    if (EPI == EPI_SWIGLU) {
      na = Wn + (size_t)item * rowb; nb = W3n + (size_t)item * rowb;
      sa = Wsz + (size_t)item * G; sb = W3sz + (size_t)item * G;
    } else {
      na = Wn + (size_t)(2 * item) * rowb; nb = na + rowb;
      sa = Wsz + (size_t)(2 * item) * G; sb = sa + G;
    }
    float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;  // [weight row][activation row]
    // software pipeline: the next tile's nibbles and (scale, zero) are in flight while the current one is consumed
    int t = half;
    bool have = t < NT && (t < KF || j < 8);
    uint4 va = make_uint4(0, 0, 0, 0), vb = va;
    __nv_bfloat162 fa = __floats2bfloat162_rn(0.f, 0.f), fb = fa;
    if (have) {
      const int k0 = t * 512 + j * 32;
      va = ldg_stream(reinterpret_cast<const uint4*>(na + (k0 >> 1)));
      vb = ldg_stream(reinterpret_cast<const uint4*>(nb + (k0 >> 1)));
      fa = __ldg(sa + (k0 >> 7));
      fb = __ldg(sb + (k0 >> 7));
    }
    while (have) {
      const int tc = t;
      const uint4 ca = va, cb = vb;
      const __nv_bfloat162 cfa = fa, cfb = fb;
      t += 2;
      have = t < NT && (t < KF || j < 8);
      if (have) {
        const int k0 = t * 512 + j * 32;
        va = ldg_stream(reinterpret_cast<const uint4*>(na + (k0 >> 1)));
        vb = ldg_stream(reinterpret_cast<const uint4*>(nb + (k0 >> 1)));
        fa = __ldg(sa + (k0 >> 7));
        fb = __ldg(sb + (k0 >> 7));
      }
      const float4* x0 = reinterpret_cast<const float4*>(xs + tc * 512) + j;
      const float4* x1 = reinterpret_cast<const float4*>(xs + K + tc * 512) + j;
      w4_dot32(ca, cfa, cb, cfb, x0, x1, tc < KF ? 16 : 8, a00, a01, a10, a11);
    }
    a00 = warp_sum(a00);
    a01 = warp_sum(a01);
    a10 = warp_sum(a10);
    a11 = warp_sum(a11);
    if (lane == 0) gemv_epilogue<EPI>(p, st, u, item, a00, a01, a10, a11);
  }
}

// ---------------------------------------------------------------------------------------------
// Dequantise up to five packed matrices (one layer's wqkv, wo, w1, w3, w2) into bf16 row-major [M, K] buffers, the layout
// of the bf16 arena, for the tensor-core GEMM of the prefill path.  One thread per 32 k of a row: one 128-bit nibble
// load, one (scale, zero) fetch, four 128-bit stores.
__global__ void __launch_bounds__(256) k_w4_dequant(WidenBatch m) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    if (i >= m.n) break;
    const int M = m.M[i], K = m.K[i], cpr = K >> 5;  // 32-k chunks per row
    const size_t n_chunks = (size_t)M * cpr;
    const uint8_t* src = m.src[i];
    const __nv_bfloat162* sz = reinterpret_cast<const __nv_bfloat162*>(src + w4_sz_offset(M, K));
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += stride) {
      const size_t row = c / cpr;
      const int k0 = (int)(c - row * cpr) * 32;
      const uint4 v = ldg_stream(reinterpret_cast<const uint4*>(src + row * (K >> 1) + (k0 >> 1)));
      const __nv_bfloat162 f = __ldg(sz + row * (K / W4_GROUP) + (k0 >> 7));
      const __nv_bfloat162 s2 = __low2bfloat162(f), z2 = __high2bfloat162(f);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      uint4* dst = reinterpret_cast<uint4*>(m.dst[i] + row * K + k0);
#pragma unroll
      for (int c4 = 0; c4 < 4; ++c4)
        dst[c4] = make_uint4(w4_deq_pair(w[c4], 0, s2, z2), w4_deq_pair(w[c4], 1, s2, z2),
                             w4_deq_pair(w[c4], 2, s2, z2), w4_deq_pair(w[c4], 3, s2, z2));
    }
  }
}

}  // namespace mvb
