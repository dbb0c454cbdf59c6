// Path C: ONE persistent kernel for a whole burst of decode positions (fast_model.py:150-163 for S = 1, all 24
// layers, + the sampler and loop bookkeeping of fast_inference_utils.py:61-120, 148-174): the kernel stays resident
// across tokens -- no launch, no host round trip and no cold start between positions.
//
//   * grid = one CTA per SM; every CTA owns a static slice of every weight matrix:
//       (K split s = cta % S, row tiles t = cta / S, + groups, ...)  chosen per matrix on the host.
//   * warp 0 = PRODUCER: walks the whole burst's byte schedule -- weight tiles via TMA (cp.async.bulk.tensor, 128B
//     swizzle) and KV-cache tiles (TMA for the bf16 cache, cp.async.bulk for fp32; K and V one stage each) into ONE
//     ring of smem stages guarded by full/empty mbarriers.  Weights do not depend on activations, so the producer never
//     waits for a grid barrier: the HBM stream keeps running across phase, layer AND token boundaries (the next token's first weight
//     tiles land while the grid is still sampling).  It issues no L2 prefetch beyond the ring: on an H100 SXM at 700 W
//     prefetching 1 to 32 tiles ahead (cp.async.bulk.prefetch.tensor while the ring is full) made batch-1 decode
//     13-68 % slower.
//   * warp 1 = MMA WARP: the weight tile [128 rows x 64 k] is the A operand, the staged activation rows (hi + lo bf16
//     halves, NB rows) the B operand of mma.sync.m16n8k16; fragments come from the 128B-swizzled tiles by ldmatrix and the
//     hi and lo products accumulate into one fp32 register tile [128 x NB/2].  At the end of a tile the warp parks the
//     accumulator in one of two shared-memory slots (acc_full / acc_empty hand-off) and goes on with the next tile.
//     (A warpgroup-wide wgmma would need four issuing warps; at N <= 32 one warp keeps pace with the weight stream.)
//   * warps 2..5 = COMPUTE: wait for the previous phase grid-wide (split arrive/wait counter with release/acquire
//     atomics), stage the activation operand into swizzled smem (RMSNorm gain / attention-merge / SiLU*mul fused
//     here), run the epilogues (accumulator slot -> red.global.add.f32 split-K accumulation), the decode attention on
//     smem KV tiles (mma.sync for the bf16 cache, online softmax per half-warp for the fp32 cache) and the
//     grid-distributed sampler.
//   * RMSNorm statistic without a full-row re-read: every CTA stages x[k-slice] * gain; the CTAs of tile group 0 add
//     their slice's sum of squares into stat[norm][row] (one red.add per row); the CONSUMER of the projection applies
//     rsqrt(stat / D + eps): attention scales q, k, v; the w2 staging scales g, u; the sampler scales the logits.
//     (x W^T) * rs == (x * rs) W^T up to fp32 rounding order.
//   * phases per layer: QKV | attention (+KV-cache append) | wo+residual | w1,w3 | w2+residual, then head, then
//     (fused mode) the sampler: every CTA ranks its own ~18 vocabulary entries against all 2562 (no sort), two more
//     grid barriers combine the kept mass and the exp-race arg-max, the utterance's owner CTA does the bookkeeping and
//     embeds the next token.
#pragma once
#include "stage1_kernels.cuh"
#include "tc.cuh"

namespace mvb {

constexpr int PC_THREADS = 192;      // producer warp + MMA warp + 4 compute warps
constexpr int PC_KV_TILE_BYTES = 16384;   // K (or V) tile of one (row, head): 64 bf16 / 32 fp32 positions; one ring stage
constexpr int PC_RPAD = 16;          // rows of the fp32 activation buffers (8 utterances x 2 CFG rows)
constexpr int PC_BKB_MAX = 12;       // k-blocks of the activation operand one CTA may own in a phase
constexpr int PC_MAX_STAGES = 12;    // ring stages PcShared has mbarriers for
constexpr int PC_MAX_CHUNKS = 64;    // per (row, head): ceil(2048 / 32) in fp32 mode
constexpr int PC_TRACE_EVENTS = 512;
// producer stall record (MVB_PC_TRACE): clock64 cycles the producer spent waiting for a free ring stage, summed over the
// launch per phase of the byte schedule; kept in the last entries of the CTA's trace row (a step stamps ~350 events)
enum PcStall { PCS_QKV, PCS_KV, PCS_WO, PCS_W13, PCS_W2, PCS_HEAD, PC_STALL_PHASES };
constexpr int PC_MAX_TILES = 128;    // attention KV tiles one CTA may own per layer
constexpr int PC_SAMP_OWN = 32;      // vocabulary entries one CTA may own in the fused sampler (ceil(V / grid))

struct AttTile {
  uint32_t off;     // byte offset of the tile inside one layer's K (or V) region
  uint32_t meta;    // npos | has_cur << 8 | unit_first << 9 | unit_last << 10 | owns_cur << 11
  uint32_t where;   // r | h << 8 | z << 16 | cache_row << 24
  int L;            // positions of the row incl. the current token
};

struct PcShared {   // small shared state behind the big buffers
  uint64_t b_full[PC_MAX_STAGES], b_empty[PC_MAX_STAGES], b_ready, acc_full[2], acc_empty[2], tab_ready;
  int n_att_tiles;
  int n_kv_tiles;                    // tiles of the table that are loaded (npos > 0): two ring stages each per layer
  // every CTA's private copy of the decode state of the batch (kept in lock-step: the same deterministic update
  // from the same arg-max in every CTA; only the owner CTA writes it back to global memory)
  int st_pos[PC_RPAD / 2], st_ngen[PC_RPAD / 2], st_done[PC_RPAD / 2], st_tok[PC_RPAD];
  // per-utterance constants of the launch (read once: every later use would cost a dependent global round trip)
  SamplingDev c_samp[PC_RPAD / 2];
  const float* c_noise[PC_RPAD / 2];
  const int* c_forced[PC_RPAD / 2];
  int c_budget[PC_RPAD / 2], c_nbase[PC_RPAD / 2], c_slot[PC_RPAD / 2];
  float o[8 * 128];                  // attention: per-half-warp partial outputs
  float m[8], l[8];
  float cur[256];                    // k, v of the current token
  float ss[PC_RPAD];                 // sum of squares of this CTA's K slice, per row
  float red[8];                      // block reductions (sampler)
  unsigned long long best[4];
  long long stall[PC_STALL_PHASES];  // producer stall cycles per phase (trace only)
  float own_ke[PC_RPAD / 2][PC_SAMP_OWN];   // sampler: kept exp-values of this CTA's vocabulary entries, per utterance
  int row_nz[PC_RPAD];
  AttTile att_tab[PC_MAX_TILES];
};

template <int NB> struct PcCfg {
  static constexpr int TILE_ROWS = 128;
  static constexpr int STAGE_BYTES = TILE_ROWS * 128;     // [TILE_ROWS x 64 k] bf16
  static constexpr int B_BYTES = PC_BKB_MAX * NB * 128;
  static constexpr int RH = NB / 2;                       // activation rows carried (hi rows; lo rows follow)
  static constexpr int ACC_LD = TILE_ROWS + 4;            // accumulator slot [RH][ACC_LD] fp32 (pad: conflict-free stores)
  static constexpr int ACC_BYTES = 2 * RH * ACC_LD * 4;   // two slots
  // ring depth: every whole stage that fits in 227 KB next to the activation operand, the accumulator slots and PcShared
  // (the 1024 B align the ring for the 128B swizzle)
  static constexpr int STAGES = (int)((227 * 1024 - 1024 - B_BYTES - ACC_BYTES - sizeof(PcShared) - 64) / STAGE_BYTES);
  static constexpr size_t SMEM = 1024 + (size_t)STAGES * STAGE_BYTES + B_BYTES + ACC_BYTES + sizeof(PcShared) + 64;
  static_assert(SMEM <= 227 * 1024, "persistent decode kernel exceeds the 227 KB shared-memory opt-in");
  static_assert(STAGES <= PC_MAX_STAGES, "PcShared has too few ring mbarriers");
  static_assert(PC_KV_TILE_BYTES == STAGE_BYTES, "a K or V tile travels as one ring stage");
  // the fused sampler's scratch (s_key, s_e) lives in the activation operand and the accumulator slots between tokens
  static_assert(2 * SAMP_PAD * sizeof(float) <= (size_t)B_BYTES + ACC_BYTES, "sampler scratch does not fit");
};

struct PcMat {     // one weight matrix kind, static decomposition
  int T;           // row tiles (of TILE_ROWS)
  int KB;          // k-blocks (of 64)
  int S;           // K splits
  int G;           // tile groups = gridDim / S
};

struct PcParams {
  int n_layer, D, F, V, H, S_max, R, n_utts, kv_fp32;
  int n_steps;     // decode positions this launch runs
  int fused;       // 1: sample in the kernel and advance the decode state (top_k == 0 only); 0: leave normalised logits
  float eps;
  PcMat m_qkv, m_o, m_w13, m_w2, m_head;
  const __nv_bfloat16* attn_norm;   // layer 0; layer l at + l * layer_stride
  const __nv_bfloat16* ffn_norm;
  const __nv_bfloat16* out_norm;
  size_t layer_stride;              // elements between consecutive layers' tensors
  const __nv_bfloat16* tok_emb;
  const __nv_bfloat16* pos_emb;
  const float* spk_proj;
  float* x;        // [RPAD, D]   residual stream (red.add target of wo / w2)
  float* qkv;      // [RPAD, 3D]  red.add target, zeroed during the wo phase
  float* gu;       // [RPAD, 2F]  g | u, red.add target, zeroed during the attention phase
  float* logits;   // [2*max_utts, V] red.add target (zero at launch; re-zeroed by the fused sampler)
  float* part_o;   // [RPAD*H*PC_MAX_CHUNKS, 128]
  float* part_ml;  // [RPAD*H*PC_MAX_CHUNKS, 2]
  float* stat;     // [2*n_layer + 1][RPAD] sums of squares of the normalised rows (attn, ffn per layer; final)
  float* samp_part;               // [RPAD/2][gridDim] kept probability mass of every CTA's vocabulary entries
  unsigned long long* samp_best;  // [2][RPAD/2] exp-race arg-max candidates (double-buffered by step parity)
  char* kv;
  size_t kv_half;  // bytes of one layer's K (or V) region
  unsigned* bar;   // grid-wide arrival counter (zero at launch)
  long long kv_rows_half;   // bf16 cache: rows (positions) of one layer's K (or V) region in tm_kv = kv_half / 256
  long long* trace;  // optional (debug): [gridDim][PC_TRACE_EVENTS] clock64 stamps of compute-thread 0 of the last step;
                     // the last PC_STALL_PHASES entries of a row: the producer's stall cycles of the whole launch
  S1State st;
};

// ---- small device helpers -------------------------------------------------------------------------
__device__ __forceinline__ void compute_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// byte offset of the 16-byte chunk holding k..k+7 of activation row `row` inside the activation operand
// (K-major, 128B swizzle, [k-block][NB rows][128 B])
template <int NB>
__device__ __forceinline__ uint32_t b_chunk_off(int kb_local, int row, int kchunk /* (k % 64) / 8 */) {
  return (uint32_t)(kb_local * (NB * 128)) + sw128_off(row, kchunk);
}

// split 8 fp32 into bf16 hi / lo and store both rows' chunks
template <int NB>
__device__ __forceinline__ void b_store8(uint8_t* B, int kb_local, int n, int kchunk, const float (&v)[8]) {
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) pack_hi_lo(v[2 * i], v[2 * i + 1], hi[i], lo[i]);
  *reinterpret_cast<uint4*>(B + b_chunk_off<NB>(kb_local, n, kchunk)) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<uint4*>(B + b_chunk_off<NB>(kb_local, NB / 2 + n, kchunk)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

struct PcSlice {   // what this CTA owns of one matrix
  int kb0, kb1, t0, nt, G;
};
__device__ __forceinline__ PcSlice pc_slice(const PcMat& m, int cta) {
  PcSlice s;
  const int sp = cta % m.S, g = cta / m.S;
  s.kb0 = (int)(((long long)sp * m.KB) / m.S);
  s.kb1 = (int)(((long long)(sp + 1) * m.KB) / m.S);
  s.G = m.G;
  s.t0 = g;
  s.nt = (g < m.G && g < m.T) ? (m.T - g + m.G - 1) / m.G : 0;
  return s;
}

// Attention work decomposition of one layer.  A unit = (activation row r, head h, split z): a contiguous run of
// KV tiles (ppc positions each) of that row's cache; every (r, h) is cut into nz <= zmax splits so that about one
// unit lands on every CTA at batch 1 while large batches get one multi-tile unit per (r, h).  Global unit ids are
// dealt round-robin to CTAs; the producer and the compute warps walk the identical sequence.
struct AttSplit {
  int tt, tps, nz;   // tiles of the row, tiles per split, number of splits
};
__device__ __forceinline__ AttSplit att_split(int L, int ppc, int zmax) {
  AttSplit a;
  a.tt = (L + ppc - 1) / ppc;
  const int zr = min(zmax, a.tt);
  a.tps = (a.tt + zr - 1) / zr;
  a.nz = (a.tt + a.tps - 1) / a.tps;
  return a;
}
// Per-step attention tile table of this CTA (identical for every layer; only the layer base pointer differs):
// built once per token by one thread, walked by the producer (KV loads) and by the compute warps.
__device__ __forceinline__ int build_att_table(const PcParams& p, const int* st_pos, const int* c_slot, int cta, int G, int ppc, int esz, AttTile* tab, int* row_nz) {
  const int zmax = max(1, G / (p.R * p.H));
  int nt = 0, base = 0;
  int id = cta;
  for (int r = 0; r < p.R; ++r) {
    const int u = c_slot[r >> 1];
    const int L = min(st_pos[r >> 1], p.S_max - 1) + 1;   // the decode state keeps pos inside the cache; clamp anyway
    const AttSplit a = att_split(L, ppc, zmax);
    row_nz[r] = a.nz;
    const int units = p.H * a.nz;
    const int cr = 2 * u + (r & 1);
    while (id < base + units) {            // this CTA's units inside row r: ids cta, cta+G, ...
      const int idx = id - base;
      const int h = idx / a.nz, z = idx - h * a.nz;
      const int t1 = min(a.tt, (z + 1) * a.tps);
      for (int t = z * a.tps; t < t1; ++t) {
        if (nt >= PC_MAX_TILES) __trap();   // fail loudly rather than drop work
        const int p0 = t * ppc;
        const int npos = min(L - 1, p0 + ppc) - p0;
        AttTile e;
        e.off = (uint32_t)((((size_t)cr * p.H + h) * p.S_max + p0) * 128 * esz);
        e.meta = (uint32_t)npos | ((p0 + ppc >= L) ? 0x100u : 0u) | ((t == z * a.tps) ? 0x200u : 0u) |
                 ((t == t1 - 1) ? 0x400u : 0u) | ((t1 == a.tt) ? 0x800u : 0u);
        e.where = (uint32_t)r | ((uint32_t)h << 8) | ((uint32_t)z << 16) | ((uint32_t)cr << 24);
        e.L = L;
        tab[nt++] = e;
      }
      id += G;
    }
    base += units;
  }
  return nt;
}

// e^x on the SFU without the denormal-range fix-up __expf carries (3 extra instructions + predicates per call);
// ex2.approx.ftz(-inf) = +0, which the attention loop relies on for masked positions.
__device__ __forceinline__ float fast_exp(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
  return y;
}

// order-preserving float <-> int32 image (for redux.sync.max on floats); -inf maps below every finite value
__device__ __forceinline__ int float_to_ordered(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_to_float(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

// acc[m][c] += W[16 m .. 16 m + 15][0 .. 63] * (hi + lo)[8 c .. 8 c + 7][0 .. 63] over one weight stage (128 rows x 64 k)
// and one k-block of the activation operand (NB rows: RH hi rows, then RH lo rows).  One warp, mma.sync.m16n8k16.
template <int NB>
__device__ __forceinline__ void pc_mma_stage(uint32_t w_base, uint32_t x_base, int lane, float (&acc)[8][NB / 16][4]) {
  constexpr int NC = NB / 16;   // n8 chunks per half
  const int q = lane >> 3, r8 = lane & 7;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t b[2 * NC][2];
#pragma unroll
    for (int g = 0; g < NB / 16; ++g) {   // rows 16 g .. 16 g + 15: two n8 chunks, both k halves
      uint32_t r[4];
      ldsm_b(x_base, 16 * g, kk, q, r8, r);
      b[2 * g][0] = r[0]; b[2 * g][1] = r[1]; b[2 * g + 1][0] = r[2]; b[2 * g + 1][1] = r[3];
    }
#pragma unroll
    for (int m = 0; m < 8; ++m) {
      uint32_t a[4];
      ldsm_a(w_base, 16 * m, kk, q, r8, a);
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        mma_bf16_16816(acc[m][c], a, b[c][0], b[c][1]);            // hi rows
        mma_bf16_16816(acc[m][c], a, b[NC + c][0], b[NC + c][1]);  // lo rows
      }
    }
  }
}

// dims 8 sub .. 8 sub + 7 of position p of an fp32 KV tile
__device__ __forceinline__ void load8s(const uint8_t* tile, int p, int sub, float (&v)[8]) {
  const float4* q = reinterpret_cast<const float4*>(tile + (size_t)p * 512 + sub * 32);
  const float4 a = q[0], b = q[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

template <bool KV_FP32, int NB>
__global__ void __launch_bounds__(PC_THREADS, 1)
k_decode_persistent(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_o,
                    const __grid_constant__ CUtensorMap tm_w1, const __grid_constant__ CUtensorMap tm_w3,
                    const __grid_constant__ CUtensorMap tm_w2, const __grid_constant__ CUtensorMap tm_head,
                    const __grid_constant__ CUtensorMap tm_kv, const PcParams p) {
  using Cfg = PcCfg<NB>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int RH = Cfg::RH;
  constexpr int STAGE_BYTES = Cfg::STAGE_BYTES;
  constexpr int TILE_ROWS = Cfg::TILE_ROWS;
  constexpr int SG = 2;   // activation chunks staged per thread per trip (3-4 were measured: the arrays spill, staging gets slower)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* ring = smem_raw + smem_pad_1024(smem_raw);
  uint8_t* Bop = ring + STAGES * STAGE_BYTES;
  float* accbuf = reinterpret_cast<float*>(Bop + Cfg::B_BYTES);   // [2][RH][ACC_LD]: MMA warp -> epilogue
  PcShared& sh = *reinterpret_cast<PcShared*>(Bop + Cfg::B_BYTES + Cfg::ACC_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cta = blockIdx.x, G = gridDim.x;
  const int esz = KV_FP32 ? 4 : 2;
  const int ppc = PC_KV_TILE_BYTES / (128 * esz);             // positions per KV tile

  if (warp == 0 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(ptx::smem_u32(sh.b_full + s), 1);
      ptx::mbar_init(ptx::smem_u32(sh.b_empty + s), 1);
    }
    ptx::mbar_init(ptx::smem_u32(&sh.b_ready), 1);
    for (int i = 0; i < 2; ++i) {
      ptx::mbar_init(ptx::smem_u32(sh.acc_full + i), 32);     // every lane of the MMA warp after its slot stores
      ptx::mbar_init(ptx::smem_u32(sh.acc_empty + i), 128);   // every compute thread after its slot loads
    }
    ptx::mbar_init(ptx::smem_u32(&sh.tab_ready), 1);
    ptx::fence_barrier_init();
  }
  // zero the activation operand once: rows >= R (hi and lo halves) must read as zero forever
  for (int i = tid; i < Cfg::B_BYTES / 16; i += PC_THREADS) reinterpret_cast<uint4*>(Bop)[i] = make_uint4(0, 0, 0, 0);
  if (tid < PC_RPAD) sh.ss[tid] = 0.f;
  if (tid < PC_STALL_PHASES) sh.stall[tid] = 0;
  ptx::fence_async_smem();
  __syncthreads();
  pdl_launch_dependents();

  const PcSlice s_qkv = pc_slice(p.m_qkv, cta), s_o = pc_slice(p.m_o, cta), s_w13 = pc_slice(p.m_w13, cta),
                s_w2 = pc_slice(p.m_w2, cta), s_head = pc_slice(p.m_head, cta);
  const int T1 = p.m_w13.T >> 1;  // w1 tiles; tiles >= T1 belong to w3

  // There is no warp 6 (PC_THREADS = 192).  Testing for it anyway makes ptxas place the producer's loop ahead of the
  // compute warps' code; with `warp == 0` alone the loop lands at the end of the kernel, and 8-utterance decode measured
  // 1.5 % slower on an H100 SXM at 700 W.
  if (warp == 0 || warp == 6) {
    // =================================== PRODUCER ===================================================
    // The whole warp walks the schedule (warp-uniform control flow and operands); one elected lane issues the TMA /
    // bulk-copy instructions.  Issuing them from a `lane == 0` branch makes the compiler wrap each UTMALDG in an
    // ELECT + 4 x R2UR.BROADCAST + vote loop, which capped one producer at a tile per ~0.25 us.
    // The ring is ONE FIFO with two consumers: the MMA warp takes the weight stages, the compute warps' attention the KV
    // stages.  So the issue order must equal the consumption order: layer l's qkv stages, then its KV tiles, then wo,
    // w1|w3, w2, then layer l+1.  Issuing a layer's KV tiles ahead of its qkv stages would deadlock: the attention
    // releases a KV stage only after the qkv multiply, and that multiply would need the ring to wrap past the held stage.
    const uint64_t pol = ptx::policy_evict_first();
    uint32_t slot = 0;
    auto acquire = [&](int phase) -> uint32_t {   // the next ring stage, once its consumer has released it
      const auto [s, ph] = ring_pos(slot, STAGES);
      ++slot;
      const uint32_t bar = ptx::smem_u32(sh.b_empty + s);
      if (p.trace == nullptr) {
        ptx::mbar_wait(bar, ph ^ 1u);
      } else {
        const long long t0 = clock64();
        ptx::mbar_wait(bar, ph ^ 1u);
        if (lane == 0) sh.stall[phase] += clock64() - t0;
      }
      return s;
    };
    auto gemm_tiles = [&](const CUtensorMap* tmA, const CUtensorMap* tmB2, int split_t, const PcSlice& sl, int layer, int phase) {
      for (int i = 0; i < sl.nt; ++i) {
        const int t = sl.t0 + i * sl.G;
        const CUtensorMap* tm = (t < split_t) ? tmA : tmB2;
        const int tt = (t < split_t) ? t : t - split_t;
        for (int kb = sl.kb0; kb < sl.kb1; ++kb) {
          const uint32_t s = acquire(phase);
          if (ptx::elect_one()) {
            const uint32_t full = ptx::smem_u32(sh.b_full + s);
            ptx::mbar_arrive_expect_tx(full, STAGE_BYTES);
            ptx::tma_load_3d_hint(ptx::smem_u32(ring + (size_t)s * STAGE_BYTES), tm, full, kb * 64, tt * TILE_ROWS, layer, pol);
          }
          __syncwarp();
        }
      }
    };
    // this CTA's KV tiles of layer l (table order), K then V as two consecutive stages -- they may straddle the ring's
    // wrap; positions < pos come from earlier steps
    auto kv_tiles = [&](int l) {
      const char* kbase = p.kv + (size_t)l * 2 * p.kv_half;
      const int n_tiles = sh.n_att_tiles;
      for (int i = 0; i < n_tiles; ++i) {
        const AttTile e = sh.att_tab[i];
        const int npos = (int)(e.meta & 0xffu);
        if (npos == 0) continue;                 // only the current position: it comes from registers
        for (int v = 0; v < 2; ++v) {            // K, V
          const uint32_t s = acquire(PCS_KV);
          if (ptx::elect_one()) {
            const uint32_t full = ptx::smem_u32(sh.b_full + s);
            const uint32_t dst = ptx::smem_u32(ring + (size_t)s * STAGE_BYTES);
            if constexpr (!KV_FP32) {
              // 64 positions x 128 dims as two 128B-swizzled [64 x 64] boxes (conflict-free ldmatrix); rows past npos are
              // older / zero cache contents and are masked by the consumer
              const int row = (int)((long long)(2 * l + v) * p.kv_rows_half + (long long)(e.off >> 8));
              ptx::mbar_arrive_expect_tx(full, PC_KV_TILE_BYTES);
              ptx::tma_load_2d(dst, &tm_kv, full, 0, row);
              ptx::tma_load_2d(dst + 8192, &tm_kv, full, 64, row);
            } else {
              const uint32_t bytes = (uint32_t)npos * 128 * esz;
              ptx::mbar_arrive_expect_tx(full, bytes);
              ptx::bulk_load(dst, kbase + (size_t)v * p.kv_half + e.off, bytes, full);
            }
          }
          __syncwarp();
        }
      }
    };
    for (int step = 0; step < p.n_steps; ++step) {
      for (int l = 0; l < p.n_layer; ++l) {
        gemm_tiles(&tm_qkv, &tm_qkv, 1 << 30, s_qkv, l, PCS_QKV);
        if (l == 0) ptx::mbar_wait(ptx::smem_u32(&sh.tab_ready), step & 1u);   // this token's tile table is built
        kv_tiles(l);
        gemm_tiles(&tm_o, &tm_o, 1 << 30, s_o, l, PCS_WO);
        gemm_tiles(&tm_w1, &tm_w3, T1, s_w13, l, PCS_W13);
        gemm_tiles(&tm_w2, &tm_w2, 1 << 30, s_w2, l, PCS_W2);
      }
      gemm_tiles(&tm_head, &tm_head, 1 << 30, s_head, 0, PCS_HEAD);
    }
    if (p.trace != nullptr && lane == 0)
      for (int i = 0; i < PC_STALL_PHASES; ++i) p.trace[(size_t)(cta + 1) * PC_TRACE_EVENTS - PC_STALL_PHASES + i] = sh.stall[i];
  } else if (warp == 1) {
    // =================================== MMA WARP ===================================================
    // The whole warp walks the schedule (waits and counters stay warp-uniform) and multiplies every weight stage of a
    // tile into registers; the finished tile goes to accumulator slot (tile_ctr & 1) for the epilogue of the compute warps.
    uint32_t slot = 0, tile_ctr = 0, bphase = 0;
    const uint32_t bop_u32 = ptx::smem_u32(Bop), ring_u32 = ptx::smem_u32(ring);
    auto gemm_phase = [&](const PcSlice& sl) {
      if (sl.nt == 0) return;
      ptx::mbar_wait(ptx::smem_u32(&sh.b_ready), bphase & 1u);   // activation operand of this phase staged
      ++bphase;
      for (int i = 0; i < sl.nt; ++i) {
        const auto [ab, aph] = ring_pos(tile_ctr, 2);
        float acc[8][NB / 16][4];
#pragma unroll
        for (int m = 0; m < 8; ++m)
#pragma unroll
          for (int c = 0; c < NB / 16; ++c)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[m][c][e] = 0.f;
        for (int kb = sl.kb0; kb < sl.kb1; ++kb) {
          const auto [s, ph] = ring_pos(slot, STAGES);
          ++slot;
          ptx::mbar_wait(ptx::smem_u32(sh.b_full + s), ph);
          pc_mma_stage<NB>(ring_u32 + s * STAGE_BYTES, bop_u32 + (uint32_t)(kb - sl.kb0) * (NB * 128), lane, acc);
          __syncwarp();                     // every lane's fragment loads of this stage are done
          if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(sh.b_empty + s));
        }
        ptx::mbar_wait(ptx::smem_u32(sh.acc_empty + ab), aph ^ 1u);   // epilogue drained this slot
        float* slot_p = accbuf + ab * (RH * Cfg::ACC_LD);
        const int r0 = lane >> 2, n0 = 2 * (lane & 3);
#pragma unroll
        for (int m = 0; m < 8; ++m)
#pragma unroll
          for (int c = 0; c < NB / 16; ++c) {
            float* d = slot_p + (8 * c + n0) * Cfg::ACC_LD + 16 * m + r0;
            d[0] = acc[m][c][0];
            d[Cfg::ACC_LD] = acc[m][c][1];
            d[8] = acc[m][c][2];
            d[Cfg::ACC_LD + 8] = acc[m][c][3];
          }
        ptx::mbar_arrive(ptx::smem_u32(sh.acc_full + ab));
        ++tile_ctr;
      }
    };
    uint32_t kv_stages = 0;
    for (int step = 0; step < p.n_steps; ++step) {
      for (int l = 0; l < p.n_layer; ++l) {
        gemm_phase(s_qkv);
        if (l == 0) {
          ptx::mbar_wait(ptx::smem_u32(&sh.tab_ready), step & 1u);   // this token's tile table is built
          kv_stages = 2u * (uint32_t)sh.n_kv_tiles;
        }
        // the layer's K, V stages belong to the attention.  Skipping them without a wait is safe: the next stage this
        // warp waits for comes after a b_ready that the compute warps publish only once the attention has drained them,
        // so no b_full barrier is ever waited on a full ring lap ahead of its producer.
        slot += kv_stages;
        gemm_phase(s_o);
        gemm_phase(s_w13);
        gemm_phase(s_w2);
      }
      gemm_phase(s_head);
    }
  } else {
    // =================================== COMPUTE WARPS ==============================================
    const int ct = tid - 64;            // 0..127
    const int cw = ct >> 5;             // 0..3
    uint32_t tile_ctr = 0, bar_idx = 0;
    uint32_t slot = 0;                  // ring position: advanced past the weight stages, consumed at the KV stages
    auto n_stages = [](const PcSlice& sl) { return (uint32_t)(sl.nt * (sl.kb1 - sl.kb0)); };
    const uint32_t st_qkv = n_stages(s_qkv), st_head = n_stages(s_head);
    const uint32_t st_post = n_stages(s_o) + n_stages(s_w13) + n_stages(s_w2);   // wo, w1|w3, w2: after the attention
    const uint32_t ring_u32 = ptx::smem_u32(ring);
    const float inv_D = 1.f / (float)p.D;
    pdl_wait();                         // state / x inputs of the previous kernels are visible
    int ev = 0;
    auto stamp = [&]() {
      if (p.trace != nullptr && ct == 0 && ev < PC_TRACE_EVENTS - PC_STALL_PHASES) p.trace[(size_t)cta * PC_TRACE_EVENTS + ev] = clock64();
      ++ev;
    };

    auto grid_arrive = [&]() {          // bar.sync orders every compute thread's writes before the release
      compute_sync();
      if (ct == 0) red_release_inc(p.bar);
      ++bar_idx;
    };
    auto grid_wait = [&]() {            // wait for arrival #bar_idx of every CTA
      if (ct == 0) wait_counter(p.bar, bar_idx * (unsigned)G);
      compute_sync();
    };
    auto b_publish = [&]() {            // generic-proxy smem writes -> visible to the tensor core
      ptx::fence_async_smem();
      compute_sync();
      if (ct == 0) ptx::mbar_arrive(ptx::smem_u32(&sh.b_ready));
    };
    // deterministic block reductions over the 128 compute threads (sampler)
    auto block_sum = [&](float v) -> float {
      v = warp_sum(v);
      if (lane == 0) sh.red[cw] = v;
      compute_sync();
      const float r = (sh.red[0] + sh.red[1]) + (sh.red[2] + sh.red[3]);
      compute_sync();
      return r;
    };
    auto block_max = [&](float v) -> float {
      v = warp_max(v);
      if (lane == 0) sh.red[cw] = v;
      compute_sync();
      const float r = fmaxf(fmaxf(sh.red[0], sh.red[1]), fmaxf(sh.red[2], sh.red[3]));
      compute_sync();
      return r;
    };
    // Activation operand <- hi/lo split of x * gain over this CTA's K range (the RMSNorm scale is applied by the
    // consumer of the projection).  The CTAs of tile group 0 (one per K split) add the slice's sum of squares to stat.
    auto stage_norm = [&](const PcSlice& sl, const __nv_bfloat16* gain, float* stat_row, bool owns_stat, bool from_emb) {
      if (sl.nt == 0) return;
      const int nchunk = (sl.kb1 - sl.kb0) * 8;
      const int total = p.R * nchunk;
      // SG chunks (3 SG loads) in flight per thread per trip; the trip count is warp-uniform (the statistic uses warp votes)
      for (int base = cw * 32; base < total; base += SG * 128) {
        const int i0 = base + lane;
        float4 la[SG], lb[SG];
        uint4 lg[SG];
#pragma unroll
        for (int j = 0; j < SG; ++j) {
          const int i = i0 + j * 128;
          if (i < total) {
            const int n = i / nchunk, c = i - n * nchunk;
            const int k = sl.kb0 * 64 + c * 8;
            lg[j] = *reinterpret_cast<const uint4*>(gain + k);
            if (!from_emb) {
              const float4* xr = reinterpret_cast<const float4*>(p.x + (size_t)n * p.D + k);
              la[j] = __ldcg(xr);
              lb[j] = __ldcg(xr + 1);
            } else {
              // first layer of a token: x = tok_emb + pos_emb (+ speaker projection on the conditioned row) straight from
              // the tables (fast_model.py:152-157) -- no grid-wide wait for the owner CTA's x rows
              const int b = n >> 1;
              const uint4 wt = *reinterpret_cast<const uint4*>(p.tok_emb + (size_t)sh.st_tok[n] * p.D + k);
              const uint4 wp = *reinterpret_cast<const uint4*>(p.pos_emb + (size_t)min(sh.st_pos[b], p.S_max - 1) * p.D + k);
              float4 sa = make_float4(0.f, 0.f, 0.f, 0.f), sb = sa;
              if ((n & 1) == 0) {
                const float* sp = p.spk_proj + (size_t)sh.c_slot[b] * p.D + k;
                sa = *reinterpret_cast<const float4*>(sp);
                sb = *reinterpret_cast<const float4*>(sp + 4);
              }
              la[j] = make_float4((bf_lo(wt.x) + bf_lo(wp.x)) + sa.x, (bf_hi(wt.x) + bf_hi(wp.x)) + sa.y,
                                  (bf_lo(wt.y) + bf_lo(wp.y)) + sa.z, (bf_hi(wt.y) + bf_hi(wp.y)) + sa.w);
              lb[j] = make_float4((bf_lo(wt.z) + bf_lo(wp.z)) + sb.x, (bf_hi(wt.z) + bf_hi(wp.z)) + sb.y,
                                  (bf_lo(wt.w) + bf_lo(wp.w)) + sb.z, (bf_hi(wt.w) + bf_hi(wp.w)) + sb.w);
            }
          }
        }
#pragma unroll
        for (int j = 0; j < SG; ++j) {
          const int i = i0 + j * 128;
          const bool act = i < total;                  // (trip counts are warp-uniform except in the last warp-trip)
          int n = 0, c = 0;
          float sq = 0.f;
          if (act) {
            n = i / nchunk; c = i - n * nchunk;
            const float4 a = la[j], b = lb[j];
            const uint4 gw = lg[j];
            float v[8] = {a.x * bf_lo(gw.x), a.y * bf_hi(gw.x), a.z * bf_lo(gw.y), a.w * bf_hi(gw.y),
                          b.x * bf_lo(gw.z), b.y * bf_hi(gw.z), b.z * bf_lo(gw.w), b.w * bf_hi(gw.w)};
            b_store8<NB>(Bop, c >> 3, n, c & 7, v);
            sq = a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w + b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
          }
          if (owns_stat) {
            // a warp's 32 consecutive chunks belong to one row (or straddle a row boundary): one smem atomic per warp
            const unsigned am = __ballot_sync(0xffffffffu, act);
            if (am != 0u) {
              const int lo_l = __ffs(am) - 1, hi_l = 31 - __clz(am);
              const int n_lo = __shfl_sync(0xffffffffu, n, lo_l), n_hi = __shfl_sync(0xffffffffu, n, hi_l);
              if (n_lo == n_hi) {
                const float s = warp_sum(sq);
                if (lane == lo_l) atomicAdd(&sh.ss[n_lo], s);
              } else if (act) {
                atomicAdd(&sh.ss[n], sq);
              }
            }
          }
        }
      }
      b_publish();
      if (owns_stat && ct < p.R) {
        atomicAdd(stat_row + ct, sh.ss[ct]);
        sh.ss[ct] = 0.f;
      }
    };
    // epilogue of this CTA's tiles: accumulator slot -> red.add into out[n][col0 + row]
    auto epilogue = [&](const PcSlice& sl, float* out, int ldo, int M, int split_t, float* out2) {
      for (int i = 0; i < sl.nt; ++i) {
        const int t = sl.t0 + i * sl.G;
        const auto [ab, aph] = ring_pos(tile_ctr, 2);
        ++tile_ctr;
        float* o = (t < split_t) ? out : out2;
        const int col0 = ((t < split_t) ? t : t - split_t) * TILE_ROWS;
        ptx::mbar_wait(ptx::smem_u32(sh.acc_full + ab), aph);
        const float* slot_p = accbuf + ab * (RH * Cfg::ACC_LD) + ct;
        float acc[RH];
#pragma unroll
        for (int n = 0; n < RH; ++n) acc[n] = slot_p[n * Cfg::ACC_LD];
        ptx::mbar_arrive(ptx::smem_u32(sh.acc_empty + ab));
        const int j = col0 + ct;
        if (j < M) {
#pragma unroll
          for (int n = 0; n < RH; ++n)
            if (n < p.R) atomicAdd(o + (size_t)n * ldo + j, acc[n]);
        }
      }
    };
    auto zero_slice = [&](float* buf, size_t n_floats) {   // this CTA's share of a buffer
      const size_t per = (n_floats / 4 + G - 1) / G;
      const size_t b = (size_t)cta * per, e = min(n_floats / 4, b + per);
      for (size_t i = b + ct; i < e; i += 128) reinterpret_cast<float4*>(buf)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    };
    // Sampler bookkeeping of decode_n_tokens / generate (utils:160-172, 212-226) for the draw of step `s_step`: append,
    // feed back, bump the position, latch end-of-audio / budget / context end.  EVERY CTA applies the same update to its
    // private copy of the state (thread b handles batch entry b); the owner CTA 2b also writes it back.
    auto finish_sample = [&](int s_step) {
      if (ct < p.n_utts && !sh.st_done[ct]) {
        const int b = ct, u = sh.c_slot[b];
        const unsigned long long best = __ldcg(p.samp_best + (size_t)(s_step & 1) * (PC_RPAD / 2) + b);
        const int tok = (int)(0xffffffffu - (unsigned)(best & 0xffffffffull));
        const int eoa = sh.c_samp[b].end_of_audio;
        const int budget = sh.c_budget[b];
        const int* forced = sh.c_forced[b];
        const int n = sh.st_ngen[b];
        const int fed = forced ? forced[n] : tok;
        const int np = sh.st_pos[b] + 1;
        const bool stop = fed == eoa || np >= p.st.block_size || n + 1 >= p.st.max_new || n + 1 >= budget;
        if (cta == 2 * b) {
          p.st.sampled_tokens[(size_t)u * p.st.max_new + n] = tok;
          p.st.gen_tokens[(size_t)u * p.st.max_new + n] = fed;
          p.st.row_tok[2 * u] = fed;
          p.st.row_tok[2 * u + 1] = fed;
          if (!stop) p.st.pos[u] = np;
          p.st.n_gen[u] = n + 1;
          if (stop) p.st.done[u] = 1;
        }
        sh.st_tok[2 * b] = fed;
        sh.st_tok[2 * b + 1] = fed;
        if (!stop) sh.st_pos[b] = np;
        sh.st_ngen[b] = n + 1;
        if (stop) sh.st_done[b] = 1;
      }
      compute_sync();
    };
    const bool owner = cta < p.R && (cta & 1) == 0;   // CTA 2b writes batch entry b's state and x rows back to global memory
    const int n_norm = 2 * p.n_layer + 1;
    if (ct < p.n_utts) {                // decode state as the host / the previous launch left it
      const int u = p.st.slot_map[ct];
      sh.c_slot[ct] = u;
      sh.c_samp[ct] = p.st.samp[u];
      sh.c_noise[ct] = p.st.noise[u];
      sh.c_forced[ct] = p.st.forced[u];
      sh.c_budget[ct] = p.st.budget[u];
      sh.c_nbase[ct] = p.st.noise_base[u];
      sh.st_pos[ct] = p.st.pos[u];
      sh.st_ngen[ct] = p.st.n_gen[u];
      sh.st_done[ct] = p.st.done[u];
      sh.st_tok[2 * ct] = p.st.row_tok[2 * u];
      sh.st_tok[2 * ct + 1] = p.st.row_tok[2 * u + 1];
    }
    compute_sync();

    for (int step = 0; step < p.n_steps; ++step) {
      ev = 0;
      stamp();
      // ---- token start: bookkeeping of the previous draw; attention tile table; the owner CTA materialises the x rows
      // (residual stream) in global memory -- they are first needed two grid barriers later (wo + residual), so nobody
      // waits for them: the first QKV operand is staged straight from the embedding tables by every CTA.
      if (step > 0 && p.fused) finish_sample(step - 1);
      if (ct == 0) {
        const int n_tiles = build_att_table(p, sh.st_pos, sh.c_slot, cta, G, ppc, esz, sh.att_tab, sh.row_nz);
        int n_kv = 0;
        for (int i = 0; i < n_tiles; ++i) n_kv += (sh.att_tab[i].meta & 0xffu) != 0u;
        sh.n_att_tiles = n_tiles;
        sh.n_kv_tiles = n_kv;
        ptx::mbar_arrive(ptx::smem_u32(&sh.tab_ready));   // release: the producer may walk the table
      }
      if (owner) {
        const int b = cta >> 1, u = sh.c_slot[b];
        const __nv_bfloat16* pe = p.pos_emb + (size_t)min(sh.st_pos[b], p.S_max - 1) * p.D;
        const __nv_bfloat16* te0 = p.tok_emb + (size_t)sh.st_tok[2 * b] * p.D;
        const __nv_bfloat16* te1 = p.tok_emb + (size_t)sh.st_tok[2 * b + 1] * p.D;
        for (int d = ct * 8; d < p.D; d += 128 * 8) {       // 8 elements per thread per trip, all loads issued together
          const uint4 wp = *reinterpret_cast<const uint4*>(pe + d);
          const uint4 w0 = *reinterpret_cast<const uint4*>(te0 + d);
          const uint4 w1 = *reinterpret_cast<const uint4*>(te1 + d);
          const float4 sa = *reinterpret_cast<const float4*>(p.spk_proj + (size_t)u * p.D + d);
          const float4 sb = *reinterpret_cast<const float4*>(p.spk_proj + (size_t)u * p.D + d + 4);
          const float pv[8] = {bf_lo(wp.x), bf_hi(wp.x), bf_lo(wp.y), bf_hi(wp.y), bf_lo(wp.z), bf_hi(wp.z), bf_lo(wp.w), bf_hi(wp.w)};
          const float t0[8] = {bf_lo(w0.x), bf_hi(w0.x), bf_lo(w0.y), bf_hi(w0.y), bf_lo(w0.z), bf_hi(w0.z), bf_lo(w0.w), bf_hi(w0.w)};
          const float t1[8] = {bf_lo(w1.x), bf_hi(w1.x), bf_lo(w1.y), bf_hi(w1.y), bf_lo(w1.z), bf_hi(w1.z), bf_lo(w1.w), bf_hi(w1.w)};
          const float sv[8] = {sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w};
          float r0[8], r1[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            r0[e] = (t0[e] + pv[e]) + sv[e];      // conditioned row: + speaker projection (fast_model.py:155-157)
            r1[e] = t1[e] + pv[e];
          }
          float4* x0 = reinterpret_cast<float4*>(p.x + (size_t)cta * p.D + d);
          float4* x1 = reinterpret_cast<float4*>(p.x + (size_t)(cta + 1) * p.D + d);
          x0[0] = make_float4(r0[0], r0[1], r0[2], r0[3]); x0[1] = make_float4(r0[4], r0[5], r0[6], r0[7]);
          x1[0] = make_float4(r1[0], r1[1], r1[2], r1[3]); x1[1] = make_float4(r1[4], r1[5], r1[6], r1[7]);
        }
      }
      compute_sync();
      stamp();

      for (int l = 0; l < p.n_layer; ++l) {
        const size_t lo_ = (size_t)l * p.layer_stride;
        float* stat_a = p.stat + (size_t)(2 * l) * PC_RPAD;
        float* stat_f = stat_a + PC_RPAD;
        // ---- QKV: operand = x * attn_norm; out: qkv (zero on entry)
        if (l > 0) grid_wait();
        stamp();
        stage_norm(s_qkv, p.attn_norm + lo_, stat_a, cta < p.m_qkv.S, l == 0);
        stamp();
        epilogue(s_qkv, p.qkv, 3 * p.D, 3 * p.D, 1 << 30, nullptr);
        stamp();
        grid_arrive();

        // ---- attention over [0, pos] + KV-cache append (fast_model.py:104-113, 220-224)
        zero_slice(p.gu, (size_t)PC_RPAD * 2 * p.F);   // free since the previous layer's w2 phase; ordered by the next arrive
        slot += st_qkv;
        grid_wait();
        stamp();
        if constexpr (!KV_FP32) {
          // ===== tensor-core attention (bf16 cache): per 64-position tile  S = K q  and  o += V^T p  as mma.sync m16n8k16 with the
          // vector operand in column 0 of the 8-wide B fragment (lanes 0..3), K / V^T blocks through ldmatrix from the
          // 128B-swizzled tiles.  q and p ride as two bf16 terms (hi + lo, 2^-17), K and V are exactly the cache contents,
          // accumulation is fp32: the same numerics class as the fp32-cache loop.  Warp w scores positions [16w, 16w+16) and
          // accumulates output dims [32w, 32w+32); every warp keeps the identical running (max, sum).
          char* kbase = p.kv + (size_t)l * 2 * p.kv_half;
          char* vbase = kbase + p.kv_half;
          uint32_t* q_hi = reinterpret_cast<uint32_t*>(sh.o);     // [64] packed pairs   (sh.o is the fp32-cache loop's merge buffer)
          uint32_t* q_lo = q_hi + 64;                             // [64]
          float* scv = reinterpret_cast<float*>(q_lo + 64);       // [64] scores of the tile
          float* qf = scv + 64;                                   // [128] fp32 q (current-token dot product)
          uint32_t* pw = reinterpret_cast<uint32_t*>(qf + 128) + cw * 64;   // per warp: [32] hi pairs | [32] lo pairs
          const int g = lane >> 2, t4 = lane & 3, mat = lane >> 3;
          float m = -INFINITY, lsum = 0.f, kcur = 0.f, vcur = 0.f;
          float oacc[2][4];
          const int n_tiles = sh.n_att_tiles;
          for (int ti = 0; ti < n_tiles; ++ti) {
            const AttTile e = sh.att_tab[ti];
            const int npos = (int)(e.meta & 0xffu);
            const bool has_cur = e.meta & 0x100u, unit_first = e.meta & 0x200u, unit_last = e.meta & 0x400u,
                       owns_cur = e.meta & 0x800u;
            const int r = e.where & 0xff, h = (e.where >> 8) & 0xff, z = (e.where >> 16) & 0xff, cr = e.where >> 24;
            const int L = e.L;
            if (unit_first) {
              const float* qrow = p.qkv + (size_t)r * 3 * p.D + h * 128;
              const float qraw = __ldcg(qrow + ct);
              const float ssr = __ldcg(stat_a + r);
              if (owns_cur) {
                kcur = __ldcg(qrow + p.D + ct);
                vcur = __ldcg(qrow + 2 * p.D + ct);
              }
              const float rsn = rsqrtf(ssr * inv_D + p.eps);      // RMSNorm scale of this row (fast_model.py:254-255)
              const float qv = qraw * (0.08838834764831845f * rsn);
              kcur *= rsn;
              vcur *= rsn;
              const float qn = __shfl_down_sync(0xffffffffu, qv, 1);
              qf[ct] = qv;
              if ((ct & 1) == 0) pack_hi_lo(qv, qn, q_hi[ct >> 1], q_lo[ct >> 1]);
              m = -INFINITY; lsum = 0.f;
#pragma unroll
              for (int i = 0; i < 4; ++i) { oacc[0][i] = 0.f; oacc[1][i] = 0.f; }
              compute_sync();                                    // q visible to every warp
            }
            if (has_cur) {
              // append the new token's k, v to the cache, rounded as the cache stores them; share them via smem
              const size_t ce = (((size_t)cr * p.H + h) * p.S_max + (L - 1)) * 128 + ct;
              const __nv_bfloat16 kb16 = __float2bfloat16_rn(kcur), vb16 = __float2bfloat16_rn(vcur);
              reinterpret_cast<__nv_bfloat16*>(kbase)[ce] = kb16;
              reinterpret_cast<__nv_bfloat16*>(vbase)[ce] = vb16;
              kcur = __bfloat162float(kb16);
              vcur = __bfloat162float(vb16);
              asm volatile("fence.proxy.async.global;" ::: "memory");   // later tokens fetch this row with TMA (async proxy)
              sh.cur[ct] = kcur;
              sh.cur[128 + ct] = vcur;
            }
            const RingPos kp = ring_pos(slot, STAGES), vp = ring_pos(slot + 1, STAGES);   // K, V stages of the tile
            if (npos > 0) {
              slot += 2;
              ptx::mbar_wait(ptx::smem_u32(sh.b_full + kp.stage), kp.phase);
              const uint32_t kt = ring_u32 + kp.stage * STAGE_BYTES;
              const uint32_t vt = ring_u32 + vp.stage * STAGE_BYTES;
              if (16 * cw < npos) {
                // ---- scores of positions [16w, 16w+16): A = K rows, B = q (hi, lo) in column 0
                // four independent accumulator chains (hi / lo terms x even / odd k-steps): the mma latency, not its issue
                // rate, is what a single warp per scheduler pays
                float c4[4][4];
#pragma unroll
                for (int i = 0; i < 4; ++i) { c4[i][0] = c4[i][1] = c4[i][2] = c4[i][3] = 0.f; }
                const int rr = 16 * cw + (lane & 7) + ((mat & 1) << 3);
#pragma unroll
                for (int k8 = 0; k8 < 8; ++k8) {
                  const int chunk = ((k8 & 3) << 1) + (mat >> 1);
                  uint32_t a[4];
                  ldsm_x4(kt + (uint32_t)((k8 >> 2) * 8192) + sw128_off(rr, chunk), a);
                  const uint32_t bh0 = lane < 4 ? q_hi[k8 * 8 + t4] : 0u, bh1 = lane < 4 ? q_hi[k8 * 8 + t4 + 4] : 0u;
                  const uint32_t bl0 = lane < 4 ? q_lo[k8 * 8 + t4] : 0u, bl1 = lane < 4 ? q_lo[k8 * 8 + t4 + 4] : 0u;
                  mma_bf16_16816(c4[(k8 & 1) * 2], a, bh0, bh1);
                  mma_bf16_16816(c4[(k8 & 1) * 2 + 1], a, bl0, bl1);
                }
                if (t4 == 0) {
                  const int p0 = 16 * cw + g;
                  scv[p0] = p0 < npos ? (c4[0][0] + c4[2][0]) + (c4[1][0] + c4[3][0]) : -INFINITY;
                  scv[p0 + 8] = p0 + 8 < npos ? (c4[0][2] + c4[2][2]) + (c4[1][2] + c4[3][2]) : -INFINITY;
                }
              } else if (lane < 16) {
                scv[16 * cw + lane] = -INFINITY;
              }
              compute_sync();                                    // all 64 scores visible: every read of K is done
              if (ct == 0) ptx::mbar_arrive(ptx::smem_u32(sh.b_empty + kp.stage));
              // ---- online softmax over the tile (identical in every warp)
              // tile max with ONE redux.sync on an order-preserving integer image of the floats (a 5-step shuffle butterfly
              // is ~150 cycles of dependent latency); the running sum stays per lane and is reduced once per unit
              const float s0 = scv[lane], s1 = scv[lane + 32];
              const float mn = fmaxf(m, ordered_to_float(__reduce_max_sync(0xffffffffu, float_to_ordered(fmaxf(s0, s1)))));
              const float mref = (mn == -INFINITY) ? 0.f : mn;
              const float corr = fast_exp(m - mref), p0v = fast_exp(s0 - mref), p1v = fast_exp(s1 - mref);
              lsum = lsum * corr + (p0v + p1v);
              m = mn;
              {
                const float n0 = __shfl_down_sync(0xffffffffu, p0v, 1), n1 = __shfl_down_sync(0xffffffffu, p1v, 1);
                if ((lane & 1) == 0) {
                  pack_hi_lo(p0v, n0, pw[lane >> 1], pw[32 + (lane >> 1)]);
                  pack_hi_lo(p1v, n1, pw[16 + (lane >> 1)], pw[48 + (lane >> 1)]);
                }
              }
              __syncwarp();
              // ---- o[32w .. 32w+32) = o * corr + V^T p : A = V^T blocks (ldmatrix.trans), B = p (hi, lo) in column 0
#pragma unroll
              for (int i = 0; i < 4; ++i) { oacc[0][i] *= corr; oacc[1][i] *= corr; }
              float olo[2][4];
#pragma unroll
              for (int i = 0; i < 4; ++i) { olo[0][i] = 0.f; olo[1][i] = 0.f; }
              const int n_k4 = (npos + 15) >> 4;
              ptx::mbar_wait(ptx::smem_u32(sh.b_full + vp.stage), vp.phase);
#pragma unroll
              for (int k4 = 0; k4 < 4; ++k4) {
                if (k4 < n_k4) {
                  const uint32_t bh0 = lane < 4 ? pw[k4 * 8 + t4] : 0u, bh1 = lane < 4 ? pw[k4 * 8 + t4 + 4] : 0u;
                  const uint32_t bl0 = lane < 4 ? pw[32 + k4 * 8 + t4] : 0u, bl1 = lane < 4 ? pw[32 + k4 * 8 + t4 + 4] : 0u;
                  const int pos = 16 * k4 + (lane & 7) + ((mat >> 1) << 3);
#pragma unroll
                  for (int mb = 0; mb < 2; ++mb) {
                    const int d0 = 32 * cw + 16 * mb;
                    const int chunk = ((d0 & 63) >> 3) + (mat & 1);
                    uint32_t a[4];
                    ldsm_x4_t(vt + (uint32_t)((d0 >> 6) * 8192) + sw128_off(pos, chunk), a);
                    mma_bf16_16816(oacc[mb], a, bh0, bh1);
                    mma_bf16_16816(olo[mb], a, bl0, bl1);
                  }
                }
              }
#pragma unroll
              for (int i = 0; i < 4; ++i) { oacc[0][i] += olo[0][i]; oacc[1][i] += olo[1][i]; }
            }
            if (npos > 0 || has_cur) compute_sync();   // V stage fully consumed; sh.cur visible
            if (npos > 0 && ct == 0) ptx::mbar_arrive(ptx::smem_u32(sh.b_empty + vp.stage));
            if (has_cur) {
              // the current token (its k, v never left the chip): every warp applies the same update to its dims
              float sd = 0.f;
#pragma unroll
              for (int i = 0; i < 4; ++i) sd = fmaf(qf[lane * 4 + i], sh.cur[lane * 4 + i], sd);
              sd = warp_sum(sd);
              const float mn = fmaxf(m, sd), corr = __expf(m - mn), pc = __expf(sd - mn);
              lsum = lsum * corr + (lane == 0 ? pc : 0.f);           // (lsum is a per-lane partial sum)
#pragma unroll
              for (int mb = 0; mb < 2; ++mb) {
                const int d = 32 * cw + 16 * mb + g;
                oacc[mb][0] = oacc[mb][0] * corr + pc * sh.cur[128 + d];
                oacc[mb][2] = oacc[mb][2] * corr + pc * sh.cur[128 + d + 8];
              }
              m = mn;
            }
            if (unit_last) {
              // every warp holds the same (m, l); output dims live in the lanes with t4 == 0 (column 0 of the C fragments)
              const size_t pidx = ((size_t)r * p.H + h) * PC_MAX_CHUNKS + z;
              if (t4 == 0) {
#pragma unroll
                for (int mb = 0; mb < 2; ++mb) {
                  const int d = 32 * cw + 16 * mb + g;
                  p.part_o[pidx * 128 + d] = oacc[mb][0];
                  p.part_o[pidx * 128 + d + 8] = oacc[mb][2];
                }
              }
              const float ltot = warp_sum(lsum);
              if (ct == 0) { p.part_ml[pidx * 2] = m; p.part_ml[pidx * 2 + 1] = ltot; }
              compute_sync();   // q / score scratch and sh.cur are reused by the next unit
            }
          }
        } else {
          // ===== fp32 cache: each half-warp runs an online softmax over its share of the tile's positions
          char* kbase = p.kv + (size_t)l * 2 * p.kv_half;
          char* vbase = kbase + p.kv_half;
          const int half = lane >> 4, sub = lane & 15;
          const int hw = cw * 2 + half;               // half-warp id 0..7
          float q[8], o[8], m = -INFINITY, lsum = 0.f, kcur = 0.f, vcur = 0.f;
          const int n_tiles = sh.n_att_tiles;
          for (int ti = 0; ti < n_tiles; ++ti) {
            const AttTile e = sh.att_tab[ti];
            const int npos = (int)(e.meta & 0xffu);
            const bool has_cur = e.meta & 0x100u, unit_first = e.meta & 0x200u, unit_last = e.meta & 0x400u,
                       owns_cur = e.meta & 0x800u;
            const int r = e.where & 0xff, h = (e.where >> 8) & 0xff, z = (e.where >> 16) & 0xff, cr = e.where >> 24;
            const int L = e.L;
            if (unit_first) {
              // ---- unit begin: one round trip for everything the unit needs from global memory
              const float* qrow = p.qkv + (size_t)r * 3 * p.D + h * 128;
              const float4 qa = __ldcg(reinterpret_cast<const float4*>(qrow + sub * 8));
              const float4 qb = __ldcg(reinterpret_cast<const float4*>(qrow + sub * 8) + 1);
              const float ssr = __ldcg(stat_a + r);
              if (owns_cur) {
                kcur = __ldcg(qrow + p.D + ct);
                vcur = __ldcg(qrow + 2 * p.D + ct);
              }
              const float rsn = rsqrtf(ssr * inv_D + p.eps);      // RMSNorm scale of this row (fast_model.py:254-255)
              const float sc = 0.08838834764831845f * rsn;        // 1/sqrt(128)
              kcur *= rsn;
              vcur *= rsn;
              q[0] = qa.x * sc; q[1] = qa.y * sc; q[2] = qa.z * sc; q[3] = qa.w * sc;
              q[4] = qb.x * sc; q[5] = qb.y * sc; q[6] = qb.z * sc; q[7] = qb.w * sc;
              m = -INFINITY; lsum = 0.f;
#pragma unroll
              for (int i = 0; i < 8; ++i) o[i] = 0.f;
            }
            // ---- one KV tile (and, on the row's last tile, the current token)
            if (has_cur) {
              // append the new token's k, v to the cache; share them via smem
              const size_t ce = (((size_t)cr * p.H + h) * p.S_max + (L - 1)) * 128 + ct;
              reinterpret_cast<float*>(kbase)[ce] = kcur;
              reinterpret_cast<float*>(vbase)[ce] = vcur;
              // the next token's KV tiles are fetched with cp.async.bulk (async proxy) inside this same launch
              asm volatile("fence.proxy.async.global;" ::: "memory");
              sh.cur[ct] = kcur;
              sh.cur[128 + ct] = vcur;
            }
            const RingPos kp = ring_pos(slot, STAGES), vp = ring_pos(slot + 1, STAGES);   // K, V stages of the tile
            if (npos > 0) {
              slot += 2;
              ptx::mbar_wait(ptx::smem_u32(sh.b_full + kp.stage), kp.phase);
              ptx::mbar_wait(ptx::smem_u32(sh.b_full + vp.stage), vp.phase);
              const uint8_t* kt = ring + (size_t)kp.stage * STAGE_BYTES;
              const uint8_t* vt = ring + (size_t)vp.stage * STAGE_BYTES;
              // each half-warp owns positions hw, hw+8, ... (hw = 2 * warp + half); two positions per trip for ILP (four per
              // trip was measured: the extra 32 live registers spill in this 255-register kernel and the phase gets 15-30 %
              // slower).  The trip count is WARP-uniform and out-of-range positions are clamped to position 0 with score -inf
              // (weight exactly 0): full-mask shuffles (no MATCH.ANY / BRA.DIV convergence checks per shuffle) and no
              // select between the dependent FMAs of the dot products.
              for (int pb = cw * 2; pb < npos; pb += 16) {
                const int pA0 = pb + half, pB0 = pA0 + 8;
                const bool vA = pA0 < npos, vB = pB0 < npos;
                const int pA = vA ? pA0 : 0, pB = vB ? pB0 : 0;
                float ka[8], kb2[8], sA = 0.f, sA1 = 0.f, sB = 0.f, sB1 = 0.f;
                load8s(kt, pA, sub, ka);
                load8s(kt, pB, sub, kb2);
#pragma unroll
                for (int i = 0; i < 8; i += 2) {
                  sA = fmaf(q[i], ka[i], sA);
                  sA1 = fmaf(q[i + 1], ka[i + 1], sA1);
                  sB = fmaf(q[i], kb2[i], sB);
                  sB1 = fmaf(q[i + 1], kb2[i + 1], sB1);
                }
                sA += sA1;
                sB += sB1;
#pragma unroll
                for (int off = 8; off > 0; off >>= 1) {   // xor offsets < 16: the reduction stays inside the 16-lane group
                  sA += __shfl_xor_sync(0xffffffffu, sA, off);
                  sB += __shfl_xor_sync(0xffffffffu, sB, off);
                }
                load8s(vt, pA, sub, ka);
                load8s(vt, pB, sub, kb2);
                sA = vA ? sA : -INFINITY;
                sB = vB ? sB : -INFINITY;
                const float mn = fmaxf(m, fmaxf(sA, sB));
                const float mref = (mn == -INFINITY) ? 0.f : mn;          // nothing valid yet: every weight below is exp(-inf) = 0
                const float corr = fast_exp(m - mref), wA = fast_exp(sA - mref), wB = fast_exp(sB - mref);
                lsum = lsum * corr + wA + wB;
#pragma unroll
                for (int i = 0; i < 8; ++i) o[i] = fmaf(o[i], corr, fmaf(wA, ka[i], wB * kb2[i]));
                m = mn;
              }
            }
            if (npos > 0 || has_cur) compute_sync();   // KV tile fully consumed; sh.cur visible
            if (npos > 0 && ct == 0) {
              ptx::mbar_arrive(ptx::smem_u32(sh.b_empty + kp.stage));
              ptx::mbar_arrive(ptx::smem_u32(sh.b_empty + vp.stage));
            }
            if (has_cur && hw == 0) {
              float sdot = 0.f;
#pragma unroll
              for (int i = 0; i < 8; ++i) sdot = fmaf(q[i], sh.cur[sub * 8 + i], sdot);
#pragma unroll
              for (int off = 8; off > 0; off >>= 1) sdot += __shfl_xor_sync(0x0000ffffu, sdot, off);
              const float mn = fmaxf(m, sdot), corr = __expf(m - mn), pw = __expf(sdot - mn);
              lsum = lsum * corr + pw;
#pragma unroll
              for (int i = 0; i < 8; ++i) o[i] = o[i] * corr + pw * sh.cur[128 + sub * 8 + i];
              m = mn;
            }
            if (unit_last) {
              // ---- unit end: merge the 8 half-warp states -> one partial (m, l, o[128]) for split z
              if (sub == 0) { sh.m[hw] = m; sh.l[hw] = lsum; }
#pragma unroll
              for (int i = 0; i < 8; ++i) sh.o[hw * 128 + sub * 8 + i] = o[i];
              compute_sync();
              {
                float M = -INFINITY;
#pragma unroll
                for (int i = 0; i < 8; ++i) M = fmaxf(M, sh.m[i]);
                float Ls = 0.f, O = 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i)
                  if (sh.m[i] > -INFINITY) {
                    const float w = __expf(sh.m[i] - M);
                    Ls += sh.l[i] * w;
                    O += sh.o[i * 128 + ct] * w;
                  }
                const size_t pidx = ((size_t)r * p.H + h) * PC_MAX_CHUNKS + z;
                p.part_o[pidx * 128 + ct] = O;
                if (ct == 0) { p.part_ml[pidx * 2] = M; p.part_ml[pidx * 2 + 1] = Ls; }
              }
              compute_sync();   // sh.o / sh.m / sh.cur are reused by the next unit
            }
          }
        }
        stamp();
        grid_arrive();

        // ---- wo + residual: operand = merged attention output (columns = this CTA's K range of heads)
        grid_wait();
        stamp();
        if (s_o.nt > 0) {
          const int nchunk = (s_o.kb1 - s_o.kb0) * 8;
          for (int i = ct; i < p.R * nchunk; i += 128) {
            const int n = i / nchunk, c = i - n * nchunk;
            const int k = s_o.kb0 * 64 + c * 8;
            const int h = k >> 7, d0 = k & 127;
            const int nch = sh.row_nz[n];
            const size_t pb = ((size_t)n * p.H + h) * PC_MAX_CHUNKS;
            float M = -INFINITY;
            float den = 0.f, v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = 0.f;
            if (nch <= 4) {
              // one round trip: (m, l) and o of every split are requested together
              float2 ml[4];
              float4 oa[4], ob[4];
#pragma unroll
              for (int z = 0; z < 4; ++z)
                if (z < nch) {
                  ml[z] = __ldcg(reinterpret_cast<const float2*>(p.part_ml + (pb + z) * 2));
                  const float4* po = reinterpret_cast<const float4*>(p.part_o + (pb + z) * 128 + d0);
                  oa[z] = __ldcg(po);
                  ob[z] = __ldcg(po + 1);
                }
#pragma unroll
              for (int z = 0; z < 4; ++z)
                if (z < nch) M = fmaxf(M, ml[z].x);
#pragma unroll
              for (int z = 0; z < 4; ++z)
                if (z < nch) {
                  const float w = __expf(ml[z].x - M);
                  den += ml[z].y * w;
                  v[0] += oa[z].x * w; v[1] += oa[z].y * w; v[2] += oa[z].z * w; v[3] += oa[z].w * w;
                  v[4] += ob[z].x * w; v[5] += ob[z].y * w; v[6] += ob[z].z * w; v[7] += ob[z].w * w;
                }
            } else {
              for (int z = 0; z < nch; ++z) M = fmaxf(M, __ldcg(p.part_ml + (pb + z) * 2));
              for (int z = 0; z < nch; ++z) {
                const float w = __expf(__ldcg(p.part_ml + (pb + z) * 2) - M);
                den += __ldcg(p.part_ml + (pb + z) * 2 + 1) * w;
                const float4* po = reinterpret_cast<const float4*>(p.part_o + (pb + z) * 128 + d0);
                const float4 a = __ldcg(po), b = __ldcg(po + 1);
                v[0] += a.x * w; v[1] += a.y * w; v[2] += a.z * w; v[3] += a.w * w;
                v[4] += b.x * w; v[5] += b.y * w; v[6] += b.z * w; v[7] += b.w * w;
              }
            }
            const float inv = 1.f / den;
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] *= inv;
            b_store8<NB>(Bop, c >> 3, n, c & 7, v);
          }
          b_publish();
        }
        stamp();
        epilogue(s_o, p.x, p.D, p.D, 1 << 30, nullptr);
        stamp();
        grid_arrive();
        zero_slice(p.qkv, (size_t)PC_RPAD * 3 * p.D);  // q, k, v were consumed by the attention phase; ordered by the next arrive

        // ---- w1 | w3: operand = x * ffn_norm; out: g | u (zero on entry)
        grid_wait();
        stamp();
        stage_norm(s_w13, p.ffn_norm + lo_, stat_f, cta < p.m_w13.S, false);
        stamp();
        epilogue(s_w13, p.gu, 2 * p.F, p.F, T1, p.gu + p.F);
        stamp();
        grid_arrive();

        // ---- w2 + residual: operand = silu(rs g) * (rs u) (fast_model.py:237, with the RMSNorm scale of the ffn input)
        grid_wait();
        stamp();
        if (s_w2.nt > 0) {
          const int nchunk = (s_w2.kb1 - s_w2.kb0) * 8;
          const int total = p.R * nchunk;
          for (int i0 = ct; i0 < total; i0 += SG * 128) {
            float4 g0[SG], g1[SG], u0[SG], u1[SG];
            float ssn[SG];
#pragma unroll
            for (int j = 0; j < SG; ++j) {
              const int i = i0 + j * 128;
              if (i < total) {
                const int n = i / nchunk, c = i - n * nchunk;
                const int k = s_w2.kb0 * 64 + c * 8;
                const float4* gp = reinterpret_cast<const float4*>(p.gu + (size_t)n * 2 * p.F + k);
                const float4* up = reinterpret_cast<const float4*>(p.gu + (size_t)n * 2 * p.F + p.F + k);
                g0[j] = __ldcg(gp); g1[j] = __ldcg(gp + 1); u0[j] = __ldcg(up); u1[j] = __ldcg(up + 1);
                ssn[j] = __ldcg(stat_f + n);
              }
            }
#pragma unroll
            for (int j = 0; j < SG; ++j) {
              const int i = i0 + j * 128;
              if (i < total) {
                const int n = i / nchunk, c = i - n * nchunk;
                const float rs = rsqrtf(ssn[j] * inv_D + p.eps);
                const float g[8] = {g0[j].x, g0[j].y, g0[j].z, g0[j].w, g1[j].x, g1[j].y, g1[j].z, g1[j].w};
                const float uu[8] = {u0[j].x, u0[j].y, u0[j].z, u0[j].w, u1[j].x, u1[j].y, u1[j].z, u1[j].w};
                float v[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                  const float ge = g[e] * rs;
                  v[e] = __fdividef(ge, 1.f + __expf(-ge)) * (uu[e] * rs);   // SiLU, 2-ulp division
                }
                b_store8<NB>(Bop, c >> 3, n, c & 7, v);
              }
            }
          }
          b_publish();
        }
        stamp();
        epilogue(s_w2, p.x, p.D, p.D, 1 << 30, nullptr);
        stamp();
        grid_arrive();
        slot += st_post;
      }
      slot += st_head;
      // ---- head: logits += (x * out_norm) . W_out^T   (rows n = batch order; scaled by the final RMSNorm below)
      float* stat_h = p.stat + (size_t)(2 * p.n_layer) * PC_RPAD;
      grid_wait();
      zero_slice(p.gu, (size_t)PC_RPAD * 2 * p.F);
      stamp();
      stage_norm(s_head, p.out_norm, stat_h, cta < p.m_head.S, false);
      stamp();
      epilogue(s_head, p.logits, p.V, p.V, 1 << 30, nullptr);
      stamp();
      grid_arrive();
      grid_wait();                        // logits (un-normalised) and the final statistic are complete
      stamp();
      const int V = p.V;
      if (!p.fused) {
        // parity / legacy-sampler mode: apply the final RMSNorm scale in place, this CTA's share of the R rows
        const int tot = p.R * V, per = (tot + G - 1) / G;
        for (int i = cta * per + ct; i < min(tot, (cta + 1) * per); i += 128) {
          const int n = i / V;
          p.logits[i] *= rsqrtf(__ldcg(stat_h + n) * inv_D + p.eps);
        }
      } else {
        // ================= grid-distributed sampler == sample() (fast_inference_utils.py:61-120), top_k = None ==========
        // CFG mix, temperature, softmax, top-p over the ASCENDING order (drop cum <= 1-p, never the last), softmax of
        // the kept entries, arg-max of probs / Exp(1).  No sort: entry i's cumulative mass is the sum of e_j over all j
        // ordered before-or-at i; every CTA evaluates it for its own ~V/grid entries against the whole vocabulary.
        // scratch [V] each: the activation operand and the accumulator slots (contiguous) are idle from the head epilogue
        // until this CTA stages the next token's qkv operand; the ring is not, the producer streams that token into it
        float* s_key = reinterpret_cast<float*>(Bop);
        float* s_e = s_key + SAMP_PAD;
        const int per = (V + G - 1) / G;
        const int i0 = cta * per, n_own = max(0, min(V, i0 + per) - i0);
        for (int b = 0; b < p.n_utts; ++b) {
          if (sh.st_done[b]) continue;
          const SamplingDev sp = sh.c_samp[b];
          const float* lc = p.logits + (size_t)(2 * b) * V;
          const float* lu = lc + V;
          const float rs_c = rsqrtf(__ldcg(stat_h + 2 * b) * inv_D + p.eps), rs_u = rsqrtf(__ldcg(stat_h + 2 * b + 1) * inv_D + p.eps);
          // CFG mix and temperature, with torch's rounding order (utils:116, :92)
          const float g = sp.guidance, omg = __fsub_rn(1.0f, sp.guidance);
          const float tdiv = fmaxf(sp.temperature, 1e-5f);
          float mx = -INFINITY;
          for (int v0 = ct; v0 < V; v0 += 12 * 128) {       // 24 loads in flight per thread per trip
            float la[12], lb[12];
#pragma unroll
            for (int i = 0; i < 12; ++i) {
              const int v = v0 + i * 128;
              if (v < V) { la[i] = __ldcg(lc + v); lb[i] = __ldcg(lu + v); }
            }
#pragma unroll
            for (int i = 0; i < 12; ++i) {
              const int v = v0 + i * 128;
              if (v < V) {
                const float k = __fdiv_rn(__fadd_rn(__fmul_rn(g, la[i] * rs_c), __fmul_rn(omg, lb[i] * rs_u)), tdiv);
                s_key[v] = k;
                mx = fmaxf(mx, k);
              }
            }
          }
          if (b == 0) stamp();
          mx = block_max(mx);
          float zs = 0.f;
          for (int v = ct; v < V; v += 128) {
            const float e = expf(s_key[v] - mx);
            s_e[v] = e;
            zs += e;
          }
          const float Z = block_sum(zs);      // (block_sum's barriers also publish s_key / s_e)
          if (b == 0) stamp();
          // own entries: warp cw takes entries cw, cw + 4, ...; lanes stride over the vocabulary
          {
            constexpr int TPW = PC_SAMP_OWN / 4;
            float ki[TPW], acc[TPW];
            int after[TPW], ii[TPW];
#pragma unroll
            for (int t = 0; t < TPW; ++t) {
              ii[t] = i0 + cw + 4 * t;
              ki[t] = (cw + 4 * t < n_own) ? s_key[ii[t]] : INFINITY;
              acc[t] = 0.f;
              after[t] = 0;
            }
            const int nt_w = (n_own > cw) ? (n_own - cw + 3) / 4 : 0;
            if (nt_w > 0) {
#pragma unroll 4
              for (int j = lane; j < V; j += 32) {
                const float kj = s_key[j], ej = s_e[j];
#pragma unroll
                for (int t = 0; t < TPW; ++t) {
                  // ascending order, ties by index (stable); bitwise predicate logic: no divergent short-circuit branches
                  const bool before = (kj < ki[t]) | ((kj == ki[t]) & (j <= ii[t]));
                  acc[t] += before ? ej : 0.f;
                  after[t] += before ? 0 : 1;
                }
              }
            }
            const bool use_p = sp.top_p > 0.f;
            const float thr = __fsub_rn(1.0f, sp.top_p);
#pragma unroll
            for (int t = 0; t < TPW; ++t) {
              const float cum = warp_sum(acc[t]);
              int na = after[t];
#pragma unroll
              for (int o2 = 16; o2 > 0; o2 >>= 1) na += __shfl_xor_sync(0xffffffffu, na, o2);
              if (lane == 0 && cw + 4 * t < n_own) {
                const bool drop = use_p && (cum / Z <= thr) && (na != 0);   // never the last (largest) entry (utils:75-77)
                sh.own_ke[b][cw + 4 * t] = drop ? 0.f : s_e[ii[t]];
              }
            }
          }
          if (b == 0) stamp();
          compute_sync();
          if (ct == 0) {
            float ps = 0.f;
            for (int t = 0; t < n_own; ++t) ps += sh.own_ke[b][t];
            p.samp_part[(size_t)b * G + cta] = ps;
          }
          compute_sync();                     // s_key / s_e are rewritten for the next utterance
        }
        // the operand's rows >= R read as zero again
        for (int i = ct; i < Cfg::B_BYTES / 16; i += 128) reinterpret_cast<uint4*>(Bop)[i] = make_uint4(0, 0, 0, 0);
        stamp();
        grid_arrive();
        grid_wait();                          // every CTA's kept mass is visible; nobody reads the logits any more
        stamp();
        zero_slice(p.logits, (size_t)p.R * V);   // hand the accumulation rows back zeroed (ordered by the next arrive)
        if (cta == 0) {
          // every RMSNorm statistic of this token has been consumed (the last one by the sampler above); the arg-max
          // slots of the PREVIOUS draw have been read by every CTA's bookkeeping (they all passed this token's barriers)
          for (int i = ct; i < n_norm * PC_RPAD; i += 128) p.stat[i] = 0.f;
          if (ct < PC_RPAD / 2) p.samp_best[(size_t)((step & 1) ^ 1) * (PC_RPAD / 2) + ct] = 0ull;
        }
        for (int b = 0; b < p.n_utts; ++b) {
          const int u = sh.c_slot[b];
          if (sh.st_done[b]) continue;
          float part = 0.f;
          for (int c = ct; c < G; c += 128) part += __ldcg(p.samp_part + (size_t)b * G + c);
          const float kept_total = block_sum(part);   // identical in every CTA (same order)
          unsigned long long best = 0ull;
          if (ct < n_own) {
            const int v = i0 + ct;
            const SamplingDev sp = sh.c_samp[b];
            const int n_gen_u = sh.st_ngen[b];
            const unsigned long long stp = (unsigned long long)n_gen_u;
            const float* nz = sh.c_noise[b];
            const float pr = sh.own_ke[b][ct] / kept_total;
            float qv;
            if (nz) {
              qv = __ldcg(nz + (size_t)(n_gen_u - sh.c_nbase[b]) * V + v);
            } else {
              const uint4 rnd = philox4x32_10(make_uint4((unsigned)v, (unsigned)stp, (unsigned)(stp >> 32), (unsigned)u),
                                              make_uint2((unsigned)sp.seed, (unsigned)(sp.seed >> 32)));
              qv = philox_exp1(rnd.x);
            }
            const float score = __fdiv_rn(pr, qv);
            // order-preserving key for non-negative floats; ties resolve to the lowest index like torch.argmax
            best = ((unsigned long long)__float_as_uint(score) << 32) | (unsigned long long)(0xffffffffu - (unsigned)v);
          }
#pragma unroll
          for (int o2 = 16; o2 > 0; o2 >>= 1) {
            const unsigned long long n2 = __shfl_xor_sync(0xffffffffu, best, o2);
            best = n2 > best ? n2 : best;
          }
          if (lane == 0) sh.best[cw] = best;
          compute_sync();
          if (ct == 0 && n_own > 0) {
            unsigned long long bb = sh.best[0];
            for (int w2 = 1; w2 < 4; ++w2) bb = sh.best[w2] > bb ? sh.best[w2] : bb;
            atomicMax(p.samp_best + (size_t)(step & 1) * (PC_RPAD / 2) + b, bb);
          }
          compute_sync();
        }
        stamp();
        grid_arrive();
        grid_wait();                          // the arg-max of every utterance is complete
      }
      stamp();
    }
    // bookkeeping of the last draw (no further position to embed)
    if (p.fused) finish_sample(p.n_steps - 1);
  }
}

}  // namespace mvb
