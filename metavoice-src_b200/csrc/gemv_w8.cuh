// Weight-only int8 stage-1 kernels (quantisation_mode="int8", fast_inference_utils.py:283-296): the int8 counterpart of
// k_gemv for decode (path A) and the per-layer widening that feeds the bf16 tensor-core GEMM for prefill (path B).
//
// int8 matrix [M, K] (K % 256 == 0; layout in include/mvb200.h, produced only by mvb200/quantize.py:pack_int8_matrix):
//   int8 [M][K] row-major, then at the next 256-byte boundary bf16 [M] row scales s.
// Function (every kernel): y_j = s_j * sum_k x_k q_jk -- fp32 sums over the exact integer weights, the scale applied once
// per output after the whole sum (== WeightOnlyInt8Linear.forward, F.linear(x, q) * s, fast_quantize.py:196-197).
#pragma once
#include "stage1_kernels.cuh"

namespace mvb {

__host__ __device__ inline size_t w8_scale_offset(int M, int K) { return ((size_t)M * K + 255) / 256 * 256; }
__host__ __device__ inline size_t w8_matrix_bytes(int M, int K) { return w8_scale_offset(M, K) + (size_t)M * 2; }

// Byte i of a word whose bytes were flipped by ^ 0x80 (so byte = q + 128) -> q as an exact fp32: prmt places the byte
// under the exponent of 2^23 (0x4B0000bb = 2^23 + q + 128, exact: the fp32 ulp at 2^23 is 1), and one fadd removes the
// bias.  Per weight: 1 PRMT + 1 FADD (+ a quarter LOP3 for the flip).
__device__ __forceinline__ float w8_f32(uint32_t flipped, int i) {
  return __uint_as_float(__byte_perm(flipped, 0x4B000000u, 0x7540 | i)) - 8388736.f;   // 2^23 + 128
}

// Position of activation k in k_gemv_w8's shared-memory layout.  In a tile of W = min(512, K - tb) values starting at
// tb = k & ~511, lane j owns k in [tb + 16 j, tb + 16 j + 16); its i-th float4 of them sits at tb + i (W / 4) + 4 j, so
// the lanes of a warp read consecutive float4 per step (no bank conflicts).
__device__ __forceinline__ int w8_perm(int k, int K) {
  const int tb = k & ~511;
  const int W = (K - tb) < 512 ? (K - tb) : 512;
  const int r = k - tb, j = r >> 4, i = (r >> 2) & 3;
  return tb + i * (W >> 2) + (j << 2) + (r & 3);
}

// 16 consecutive k of two weight rows (va, vb: one 128-bit load each) against the two CFG activation rows (x0, x1:
// float4 c of the lane at x[c * xstride]).  Sequential fp32 fmas in k order.
__device__ __forceinline__ void w8_dot16(const uint4& va, const uint4& vb, const float4* x0, const float4* x1, int xstride,
                                         float& a00, float& a01, float& a10, float& a11) {
  const uint32_t wa[4] = {va.x ^ 0x80808080u, va.y ^ 0x80808080u, va.z ^ 0x80808080u, va.w ^ 0x80808080u};
  const uint32_t wb[4] = {vb.x ^ 0x80808080u, vb.y ^ 0x80808080u, vb.z ^ 0x80808080u, vb.w ^ 0x80808080u};
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float4 p = x0[c * xstride], q = x1[c * xstride];
    const float xp[4] = {p.x, p.y, p.z, p.w}, xq[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float qa = w8_f32(wa[c], e), qb = w8_f32(wb[c], e);
      a00 = fmaf(qa, xp[e], a00);
      a01 = fmaf(qa, xq[e], a01);
      a10 = fmaf(qb, xp[e], a10);
      a11 = fmaf(qb, xq[e], a11);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// k_gemv's contract (GemvP, the RMSNorm prologue, the four epilogues, gridDim.y = utterances) over int8 matrices: p.W (and
// p.W3 for EPI_SWIGLU) point at int8 matrices.  A warp owns one item, as in k_gemv (rows 2i, 2i + 1, or w1 row i and w3
// row i).  K is cut into NT = ceil(K / 512) tiles of 512 (a trailing one of 256 when K % 512 == 256); per tile lane j
// streams 16 k of each row with one 128-bit load per row (lanes 0-15 take the trailing 256-wide tile) and loads the next
// tile while it consumes the current one.  Per output a lane's fp32 sum runs over at most 16 NT products in k order, a
// 5-level butterfly adds the 32 lanes, and lane 0 multiplies by the row's bf16 scale (w1's for the gate, w3's for the up
// projection) before the epilogue.
// Memory pipeline as in k_gemv_w4: before griddepcontrol.wait every warp asks L2 for all the rows it will stream
//, so the matrix is in flight while the previous kernel drains.
template <int EPI>
__global__ void __launch_bounds__(256, 2) k_gemv_w8(GemvP p, S1State st) {
  extern __shared__ float xs[];  // [2][K] in the w8_perm layout
  __shared__ float red[16];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = p.K;
  const int n_items = (EPI == EPI_SWIGLU) ? p.M : (p.M >> 1);
  const uint8_t* Wq = reinterpret_cast<const uint8_t*>(p.W);
  const __nv_bfloat16* Ws = reinterpret_cast<const __nv_bfloat16*>(Wq + w8_scale_offset(p.M, K));
  const uint8_t* W3q = reinterpret_cast<const uint8_t*>(p.W3);
  const __nv_bfloat16* W3s = EPI == EPI_SWIGLU ? reinterpret_cast<const __nv_bfloat16*>(W3q + w8_scale_offset(p.M, K)) : nullptr;
  pdl_launch_dependents();
  {
    // lane n of a warp prefetches the warp's n-th item (the loop below visits the same items in the same order)
    const int item = blockIdx.x * 8 + warp + lane * gridDim.x * 8;
    if (item < n_items) {
      if (EPI == EPI_SWIGLU) {
        l2_prefetch(Wq + (size_t)item * K, K);
        l2_prefetch(W3q + (size_t)item * K, K);
      } else {
        l2_prefetch(Wq + (size_t)(2 * item) * K, 2 * (size_t)K);
      }
    }
  }
  pdl_wait();  // activations written by the previous kernel are now visible

  const int u = st.slot_map[blockIdx.y];
  gemv_prologue(p, 2 * u, xs, red, [K](int k) { return w8_perm(k, K); });

  const int KF = K >> 9;                               // full 512-wide tiles
  const int NT = KF + ((K & 511) != 0 ? 1 : 0);        // plus one trailing 256-wide tile
  for (int item = blockIdx.x * 8 + warp; item < n_items; item += gridDim.x * 8) {
    const uint8_t *ra, *rb;
    int ja, jb;                                        // rows of the scales
    if (EPI == EPI_SWIGLU) {
      ra = Wq + (size_t)item * K; rb = W3q + (size_t)item * K;
      ja = jb = item;
    } else {
      ra = Wq + (size_t)(2 * item) * K; rb = ra + K;
      ja = 2 * item; jb = ja + 1;
    }
    float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;  // [weight row][activation row]
    int t = 0;
    bool have = NT > 0 && (KF > 0 || lane < 16);
    uint4 va = make_uint4(0, 0, 0, 0), vb = va;
    if (have) {
      va = ldg_stream(ra + lane * 16);
      vb = ldg_stream(rb + lane * 16);
    }
    while (have) {
      const int tc = t;
      const uint4 ca = va, cb = vb;
      ++t;
      have = t < NT && (t < KF || lane < 16);
      if (have) {
        const int k0 = t * 512 + lane * 16;
        va = ldg_stream(ra + k0);
        vb = ldg_stream(rb + k0);
      }
      const float4* x0 = reinterpret_cast<const float4*>(xs + tc * 512) + lane;
      const float4* x1 = reinterpret_cast<const float4*>(xs + K + tc * 512) + lane;
      w8_dot16(ca, cb, x0, x1, tc < KF ? 32 : 16, a00, a01, a10, a11);
    }
    a00 = warp_sum(a00);
    a01 = warp_sum(a01);
    a10 = warp_sum(a10);
    a11 = warp_sum(a11);
    if (lane == 0) {
      const float sa = bf16_to_f32(Ws[ja]), sb = bf16_to_f32(EPI == EPI_SWIGLU ? W3s[jb] : Ws[jb]);
      gemv_epilogue<EPI>(p, st, u, item, a00 * sa, a01 * sa, a10 * sb, a11 * sb);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Widen up to five int8 matrices (one layer's wqkv, wo, w1, w3, w2, or lm_head once at create) to bf16 row-major [M, K]
// buffers holding q exactly (|q| <= 128 fits bf16's 8-bit significand), the operand of the tensor-core GEMM, whose
// epilogue applies the row scales.  One thread per 16 k of a row: one 128-bit load, two 128-bit stores.
__global__ void __launch_bounds__(256) k_w8_widen(WidenBatch m) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    if (i >= m.n) break;
    const int K = m.K[i];
    const size_t n_chunks = (size_t)m.M[i] * K / 16;   // 16-k chunks, row-major
    const uint8_t* src = m.src[i];
    uint4* dst = reinterpret_cast<uint4*>(m.dst[i]);
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += stride) {
      const uint4 v = ldg_stream(src + c * 16);
      const uint32_t w[4] = {v.x ^ 0x80808080u, v.y ^ 0x80808080u, v.z ^ 0x80808080u, v.w ^ 0x80808080u};
      uint32_t o[8];
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const __nv_bfloat162 lo = __floats2bfloat162_rn(w8_f32(w[h], 0), w8_f32(w[h], 1));
        const __nv_bfloat162 hi = __floats2bfloat162_rn(w8_f32(w[h], 2), w8_f32(w[h], 3));
        o[2 * h] = *reinterpret_cast<const uint32_t*>(&lo);
        o[2 * h + 1] = *reinterpret_cast<const uint32_t*>(&hi);
      }
      dst[2 * c] = make_uint4(o[0], o[1], o[2], o[3]);
      dst[2 * c + 1] = make_uint4(o[4], o[5], o[6], o[7]);
    }
  }
}

}  // namespace mvb
