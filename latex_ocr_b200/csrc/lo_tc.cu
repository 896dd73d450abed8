// wgmma + TMA kernels (sm_90a): the K-major "NT" GEMM, the persistent NHWC 3x3 implicit-GEMM convolution (forward and
// data gradient) and the weight gradient / "TN" GEMM.
//
//   D[128 x NT] (registers, fp32) += A[128 x 64] (smem, bf16, SWIZZLE_128B) * B[NT x 64]^T (smem, bf16, SWIZZLE_128B)
//
// Warp roles, all three kernels: warps 0..7 = two consumer warpgroups (warpgroup g owns rows [64g, 64g+64) of the tile:
// wgmma into registers, then the epilogue straight from the accumulators), warp 8 = A-tile TMA producer, warp 9 = B-tile
// TMA producer, over a 3-8 stage mbarrier ring.
//   tc_gemm_kernel    C = A W^T (+ bias, ReLU, accumulate, split-K atomics): one 128 x NT tile per CTA; 2-D maps over the
//                     K-major rows of A and W.  Option conv_mc: a CTA pair shares the A tile by multicast.
//   tc_conv_p_kernel  one CTA per SM walks over output tiles.  A tiles: a 4-D map over the NHWC feature map {C, W, H, N}
//                     with box {64, BW, BH, 1} (BW*BH = 128 output positions); tap (r,s) is a coordinate shift and the
//                     halo / zero padding falls out of TMA's out-of-bounds zero fill — no im2col buffer, no predicates.
//                     B tiles are rows of the [Cout][9*Cin] weight matrix.
//   tc_wgrad_kernel   dW = dY^T (*) X and the TN GEMMs, both operands MN-major.
#include <cuda.h>

#include <mutex>
#include <unordered_map>

#include "lo_common.cuh"
#include "lo_ptx.cuh"
#include "lo_wgmma.cuh"

namespace lo {

// ------------------------------------------------------------------------------------------------
// PTX wrappers (strings follow cute/arch/copy_sm90_tma.hpp, cutlass/arch/barrier.h)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                   smem_u32(dst)),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_load_2d_hint(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// multicast variant: the box lands at the same CTA-relative offset in every CTA of `mask` and completes on each one's mbarrier
__device__ __forceinline__ void tma_load_2d_mc(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%4, %5}], [%2], %3;" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1)
      : "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster (may be this CTA)
__device__ __forceinline__ void mbar_arrive_cta(uint64_t* bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// K-major, SWIZZLE_128B wgmma shared-memory descriptor (cute::GMMA::GmmaDescriptor): rows of 128 B, 8-row groups
// 1024 B apart (SBO), LBO unused for swizzled K-major (=1), layout type 1 (SWIZZLE_128B).  Tiles start 1024-aligned.
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);          // start address   bits [0,14)
  d |= (uint64_t)1 << 16;                           // leading byte offset (16 B units) bits [16,30)
  d |= (uint64_t)(1024 >> 4) << 32;                 // stride byte offset  bits [32,46)
  d |= (uint64_t)1 << 62;                           // SWIZZLE_128B        bits [62,64)
  return d;
}

// the NT GEMM C[M][N] = A[M][K] W[N][K]^T
struct TcParams {
  int M, N, K;
  // epilogue
  const float* bias;
  void* out;
  int64_t ldc;
  int out_f32, accumulate, relu;
  int kb_per_split, atomic;   // split-K over gridDim.z: fp32 atomics onto `out` (bias added by split 0)
  int w_evict_last;           // keep the B (weight) tiles in L2: the per-step decoder GEMMs re-read them every step
  long long* dbg;             // optional: clock64 stamps of CTA (0,0,0) at the pipeline milestones (lo_debug_buffer)
};

// the 3x3 convolution: GEMM view M = output positions, N = Cout, K = 9 * Cin
struct ConvParams {
  int N, K;
  int Cin, pad, Ho, Wo;                 // output H, W
  int BW, BH, tiles_w, tiles_h;         // position box (BW * BH = 128) and boxes per output row / column
  const float* bias;
  const bf16* mask;                     // optional: outputs where mask <= 0 are 0 (the data gradient's ReLU mask)
  bf16* out;
  int64_t ldc;
  int relu;
};

constexpr int TC_BM = 128, TC_BK = 64;
constexpr int TC_CWARPS = 8;                          // two consumer warpgroups
constexpr int TC_THREADS = (TC_CWARPS + 2) * 32;      // + warp 8: A-tile TMA producer, warp 9: B-tile TMA producer

template <int NT, int STAGES>
struct TcSmem {
  static constexpr int A_BYTES = TC_BM * TC_BK * 2;      // 16 KB
  static constexpr int B_BYTES = NT * TC_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

// One K block (64 wide) of a consumer warpgroup: its 64 rows of the A stage (rows 64 * wg.., 8 KB apart) times the B stage.
template <int NT>
__device__ __forceinline__ void tc_mma_kblock(float* acc, uint32_t sa, uint32_t sb, bool first) {
  const uint64_t da = make_kmajor_sw128_desc(sa), db = make_kmajor_sw128_desc(sb);
#pragma unroll
  for (int k = 0; k < TC_BK / 16; k++)
    // advance 16 elements (32 B) along K inside the 128 B swizzle row: +2 in the 16 B-unit address field
    Wgmma<NT, 0, 0>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (first && k == 0) ? 0u : 1u);
}

// bias (+ReLU) epilogue of two adjacent accumulator columns of one output row, written to bf16 or fp32;
// `atomic` adds onto fp32 (split-K partial sums)
__device__ __forceinline__ void tc_store_pair(const TcParams& p, int64_t off, float f0, float f1) {
  if (p.atomic) {
    float* o = reinterpret_cast<float*>(p.out) + off;
    atomicAdd(o, f0);
    atomicAdd(o + 1, f1);
  } else if (p.out_f32) {
    float2* o = reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + off);
    if (p.accumulate) { const float2 old = *o; f0 += old.x; f1 += old.y; }
    if (p.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
    *o = make_float2(f0, f1);
  } else {
    uint32_t* o = reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(p.out) + off);
    if (p.accumulate) { const uint32_t old = *o; f0 += __uint_as_float(old << 16); f1 += __uint_as_float(old & 0xffff0000u); }
    if (p.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
    __nv_bfloat162 h = __floats2bfloat162_rn(f0, f1);
    *o = *reinterpret_cast<uint32_t*>(&h);
  }
}

// MC = 1: the two CTAs of a (2,1,1) cluster compute neighbouring N tiles of the SAME 128-row A tile; each loads one
// 64-row half of A and multicasts it to both (halves the L2 -> SM traffic of A).  mapA then describes 64-row boxes.
template <int NT, int STAGES, int MC>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_gemm_kernel(const __grid_constant__ CUtensorMap mapA,
                                                                 const __grid_constant__ CUtensorMap mapB, TcParams p) {
  using SM = TcSmem<NT, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * SM::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  __shared__ __align__(16) float s_bias[NT];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * NT;
  const int m0 = blockIdx.y * TC_BM;
  const int KB_all = p.K / TC_BK;
  const int kb0 = blockIdx.z * p.kb_per_split;
  const int KB = min(KB_all, kb0 + p.kb_per_split) - kb0;      // K blocks of this split

  const bool dbg = p.dbg && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0;
  if (dbg && threadIdx.x == 0) p.dbg[0] = clock64();
  if (warp == TC_CWARPS && lane == 0) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    for (int s = 0; s < STAGES; s++) {
      mbar_init(full_bar + s, 2);                 // two producer threads (A tiles / B tiles)
      mbar_init(empty_bar + s, MC ? 2 * TC_CWARPS : TC_CWARPS);   // MC: the slot is also written by the peer -> both CTAs' consumers release it
    }
    fence_barrier_init();
  }
  pdl_wait();          // everything above touched only shared memory / kernel parameters
  pdl_trigger();
  if (MC) cluster_sync_all(); else __syncthreads();   // peer barriers must be initialised before any multicast lands
  const uint32_t crank = MC ? cluster_ctarank() : 0;
  if (dbg && threadIdx.x == 0) p.dbg[1] = clock64();

  if (warp == TC_CWARPS) {
    if (lane == 0) {
      // ===== TMA producer, A tiles =====
      for (int kb = 0; kb < KB; kb++) {
        const int s = kb % STAGES;
        const uint32_t ph = (kb / STAGES) & 1;
        mbar_wait(empty_bar + s, ph ^ 1);
        uint8_t* sa = smem + s * SM::STAGE_BYTES;
        mbar_expect_tx(full_bar + s, SM::A_BYTES);
        const int kg = kb0 + kb;
        if (MC)        // my half of the tile, delivered to both CTAs
          tma_load_2d_mc(sa + crank * (SM::A_BYTES / 2), &mapA, full_bar + s, kg * TC_BK, m0 + (int)crank * (TC_BM / 2), (uint16_t)3);
        else
          tma_load_2d(sa, &mapA, full_bar + s, kg * TC_BK, m0);
        if (dbg && kb == 0) p.dbg[2] = clock64();
        if (dbg && kb < 40) p.dbg[64 + kb] = clock64();          // A-producer: TMA of K block kb issued
      }
      if (dbg) p.dbg[3] = clock64();
    }
    __syncwarp();
  } else if (warp == TC_CWARPS + 1) {
    if (lane == 0) {
      // ===== TMA producer, B tiles (weights) =====
      const uint64_t polB = p.w_evict_last ? l2_policy_evict_last() : l2_policy_evict_normal();
      for (int kb = 0; kb < KB; kb++) {
        const int s = kb % STAGES;
        const uint32_t ph = (kb / STAGES) & 1;
        mbar_wait(empty_bar + s, ph ^ 1);
        uint8_t* sb = smem + s * SM::STAGE_BYTES + SM::A_BYTES;
        mbar_expect_tx(full_bar + s, SM::B_BYTES);
        tma_load_2d_hint(sb, &mapB, full_bar + s, (kb0 + kb) * TC_BK, n0, polB);
      }
    }
    __syncwarp();
  } else {
    // ===== consumers: warpgroup wg accumulates rows [64 wg, 64 wg + 64) of the tile =====
    const int wg = warp >> 2;
    for (int c = threadIdx.x; c < NT; c += TC_CWARPS * 32)
      s_bias[c] = (p.bias && blockIdx.z == 0 && n0 + c < p.N) ? __ldg(p.bias + n0 + c) : 0.f;
    asm volatile("bar.sync 1, 256;" ::: "memory");
    float acc[NT / 2];
    for (int kb = 0; kb < KB; kb++) {
      const int s = kb % STAGES;
      const uint32_t ph = (kb / STAGES) & 1;
      mbar_wait(full_bar + s, ph);
      if (dbg && threadIdx.x == 0 && kb == 0) p.dbg[4] = clock64();
      if (dbg && threadIdx.x == 0 && kb < 40) p.dbg[16 + kb] = clock64();          // consumer: K block kb landed
      const uint32_t sa = smem_u32(smem + s * SM::STAGE_BYTES);
      wgmma_fence();
      tc_mma_kblock<NT>(acc, sa + wg * (SM::A_BYTES / 2), sa + SM::A_BYTES, kb == 0);
      wgmma_commit();
      wgmma_wait0();
      wgmma_acc_fence<NT / 2>(acc);
      __syncwarp();
      if (lane == 0) {
        if (MC) { mbar_arrive_cta(empty_bar + s, 0); mbar_arrive_cta(empty_bar + s, 1); }   // frees the slot in BOTH CTAs
        else mbar_arrive(empty_bar + s);
      }
    }
    if (dbg && threadIdx.x == 0) p.dbg[5] = clock64();
    // ===== epilogue from the accumulators (layout: lo_wgmma.cuh) =====
    const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int row = rbase + 8 * h;
      if (m0 + row >= p.M) continue;
      const int64_t row_off = (int64_t)(m0 + row) * p.ldc;
#pragma unroll
      for (int i = 0; i < NT / 8; i++) {
        if (n0 + 8 * i >= p.N) continue;       // 8-column groups: columns up to roundup8(N) are written (ldc allows it)
        const int c = 8 * i + cq;
        tc_store_pair(p, row_off + n0 + c, acc[4 * i + 2 * h] + s_bias[c], acc[4 * i + 2 * h + 1] + s_bias[c + 1]);
      }
    }
    if (dbg && threadIdx.x == 0) p.dbg[6] = clock64();
  }
  if (MC) cluster_sync_all();   // a CTA may not exit while its peer can still multicast into it or arrive on its barriers
  if (dbg && threadIdx.x == 0) p.dbg[7] = clock64();
}

// ------------------------------------------------------------------------------------------------
// Persistent 3x3 convolution (forward and data gradient): one CTA per SM walks over output tiles of MT x 128 positions x NT
// channels.  The TMA ring runs ahead across tile boundaries, so the next tile's operands stream in while the consumer
// warpgroups run the epilogue of the current one.  NT = 256 for the 256/512-channel layers: per 64-wide K block a CTA
// pulls 16 KB of A + 32 KB of B from L2 for 4.2 MFLOP = 85 FLOP per L2 byte (128 x 128 tiles: 64).
// ------------------------------------------------------------------------------------------------
template <int NT, int STAGES, int MT>
struct TcPSmem {
  static constexpr int A_BYTES = TC_BM * TC_BK * 2;              // one 128-position sub-tile
  static constexpr int B_BYTES = NT * TC_BK * 2;
  static constexpr int STAGE_BYTES = MT * A_BYTES + B_BYTES;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/ + 2 * NT * 4 /*bias, double buffered*/;
};

// MT = 2 (layers with <= 128 output channels): a CTA tile is TWO 128-position sub-tiles that share every weight (B) stage —
// FLOP per byte of A equals N in an implicit GEMM, so with N <= 128 the B stage is as large as an A tile and sharing it
// raises the FLOP per L2 byte from 64 to 87 (N = 128) / 43 to 52 (N = 64).
template <int NT, int STAGES, int MT>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_conv_p_kernel(const __grid_constant__ CUtensorMap mapA,
                                                                 const __grid_constant__ CUtensorMap mapB, ConvParams p, int ntiles_n,
                                                                 int total_tiles, int mtiles) {
  using SM = TcPSmem<NT, STAGES, MT>;
  static_assert(MT * NT <= 256, "accumulator registers");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * SM::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  float* s_bias = reinterpret_cast<float*>(smem + STAGES * SM::STAGE_BYTES + 256);      // [2][NT]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int KB = p.K / TC_BK;
  const int cpb = p.Cin / TC_BK;
  const int per_img = p.tiles_w * p.tiles_h;

  if (warp == TC_CWARPS && lane == 0) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    for (int s = 0; s < STAGES; s++) {
      mbar_init(full_bar + s, 2);                // A producer + B producer
      mbar_init(empty_bar + s, TC_CWARPS);       // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  pdl_wait();
  pdl_trigger();
  __syncthreads();

  if (warp == TC_CWARPS) {
    if (lane == 0) {
      // ===== TMA producer, A tiles (implicit im2col: tap = coordinate shift, halo = out-of-bounds zero fill) =====
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int mt0 = (tile / ntiles_n) * MT;
        const int nsub = min(MT, mtiles - mt0);
        int img[MT], h0[MT], w0[MT];
#pragma unroll
        for (int j = 0; j < MT; j++) {
          const int mt = min(mt0 + j, mtiles - 1);
          img[j] = mt / per_img;
          const int rem = mt % per_img;
          h0[j] = (rem / p.tiles_w) * p.BH;
          w0[j] = (rem % p.tiles_w) * p.BW;
        }
        for (int kb = 0; kb < KB; kb++, it++) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait(empty_bar + s, ph ^ 1);
          mbar_expect_tx(full_bar + s, (uint32_t)nsub * SM::A_BYTES);
          const int tap = kb / cpb, cb = kb % cpb;
          const int r = tap / 3, q = tap % 3;
#pragma unroll
          for (int j = 0; j < MT; j++)
            if (j < nsub)
              tma_load_4d(smem + s * SM::STAGE_BYTES + j * SM::A_BYTES, &mapA, full_bar + s, cb * TC_BK, w0[j] + q - p.pad,
                          h0[j] + r - p.pad, img[j]);
        }
      }
    }
    __syncwarp();
  } else if (warp == TC_CWARPS + 1) {
    if (lane == 0) {
      // ===== TMA producer, B tiles (weights: re-read by every CTA -> keep them in L2) =====
      const uint64_t polB = l2_policy_evict_last();
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n0 = (tile % ntiles_n) * NT;
        for (int kb = 0; kb < KB; kb++, it++) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait(empty_bar + s, ph ^ 1);
          mbar_expect_tx(full_bar + s, SM::B_BYTES);
          tma_load_2d_hint(smem + s * SM::STAGE_BYTES + MT * SM::A_BYTES, &mapB, full_bar + s, kb * TC_BK, n0, polB);
        }
      }
    }
    __syncwarp();
  } else {
    // ===== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of every sub-tile =====
    const int wg = warp >> 2;
    const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    const bool use_mask = p.mask != nullptr;
    uint32_t it = 0, lt = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, lt++) {
      const int n0 = (tile % ntiles_n) * NT;
      const int mt0 = (tile / ntiles_n) * MT;
      const int nsub = min(MT, mtiles - mt0);
      float* sb = s_bias + (lt & 1) * NT;        // double buffered: a slower thread may still read the previous tile's
      for (int c = threadIdx.x; c < NT; c += TC_CWARPS * 32) sb[c] = (p.bias && n0 + c < p.N) ? __ldg(p.bias + n0 + c) : 0.f;
      asm volatile("bar.sync 1, 256;" ::: "memory");
      float acc[MT][NT / 2];
      for (int kb = 0; kb < KB; kb++, it++) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(full_bar + s, ph);
        const uint32_t sa = smem_u32(smem + s * SM::STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < MT; j++)
          // issued for every sub-tile, also the missing last one of an odd tile count (its slot holds stale data; that
          // accumulator is never stored): a predicate here makes ptxas serialise the warpgroup MMAs
          tc_mma_kblock<NT>(acc[j], sa + j * SM::A_BYTES + wg * (SM::A_BYTES / 2), sa + MT * SM::A_BYTES, kb == 0);
        wgmma_commit();
        wgmma_wait0();
#pragma unroll
        for (int j = 0; j < MT; j++) wgmma_acc_fence<NT / 2>(acc[j]);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar + s);
      }
#pragma unroll
      for (int j = 0; j < MT; j++) {
        if (j >= nsub) continue;
        const int mt = mt0 + j;
        const int img = mt / per_img, rem = mt % per_img;
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int row = rbase + 8 * h;
          const int hh = (rem / p.tiles_w) * p.BH + row / p.BW, ww = (rem % p.tiles_w) * p.BW + row % p.BW;
          if (hh >= p.Ho || ww >= p.Wo) continue;
          const int64_t row_off = (((int64_t)img * p.Ho + hh) * p.Wo + ww) * p.ldc;
#pragma unroll
          for (int i = 0; i < NT / 8; i++) {
            if (n0 + 8 * i >= p.N) continue;
            const int c = 8 * i + cq;
            float f0 = acc[j][4 * i + 2 * h] + sb[c], f1 = acc[j][4 * i + 2 * h + 1] + sb[c + 1];
            if (p.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
            if (use_mask) {
              const uint32_t w = *reinterpret_cast<const uint32_t*>(p.mask + row_off + n0 + c);
              if (!(__uint_as_float(w << 16) > 0.f)) f0 = 0.f;
              if (!(__uint_as_float(w & 0xffff0000u) > 0.f)) f1 = 0.f;
            }
            __nv_bfloat162 hv = __floats2bfloat162_rn(f0, f1);
            *reinterpret_cast<__nv_bfloat162*>(p.out + row_off + n0 + c) = hv;
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Weight gradient on wgmma:  dW[co][tap][ci] += sum_p dY[p][co] * X[p + tap][ci]
// GEMM view: M = co (128), N = ci (NT), K = output positions.  Both operands are "MN-major" (the channel index is
// contiguous in NHWC), which wgmma takes directly (transpose flags): smem tile = [KP positions][64 channels] (one TMA
// box, SWIZZLE_128B), descriptor LBO = distance between 64-channel boxes, SBO = 1024 B (8 positions), 16 positions
// (2048 B) per MMA.  KP = 128 positions per K block, or 64 for the 128 x 256 tiles (16 KB of dY + 32 KB of X per
// stage, four stages): the host then cuts every 128-position box into two 64-position boxes in the same row-major order and
// doubles the split length, so each output element sees the same sequence of k16 MMAs.  grid: (co tiles * ci tiles,
// 9 taps, K splits); the splits add their partial sums onto dW with fp32 atomics, or — option "deterministic" — form one
// cluster (<= 8) whose rank 0 adds them in split order and alone adds the result.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t make_mnmajor_sw128_desc(uint32_t saddr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;   // next 64-element block along M/N
  d |= (uint64_t)(1024 >> 4) << 32;                   // next 8 rows along K
  d |= (uint64_t)1 << 62;                             // SWIZZLE_128B
  return d;
}

struct WgParams {
  int Cin, Cout, Ho, Wo, pad;
  int BW, BH, tiles_w, tiles_h, kstages, per_split, ci_tiles;
  float* dw;
  int plain;          // 1: plain C[M][N] += A[K][M]^T B[K][N] (2-D maps; Cout = M, Cin = N, tap ignored)
                      // 2: the same, batched over blockIdx.y (3-D maps {M|N, K, batch}; C of batch b at dw + b * batch_c)
  int64_t ldc;
  int64_t batch_c;
  int ordered;        // 1: the K splits of a tile are one cluster, summed in split order (option "deterministic")
};

template <int NT, int KP, int STAGES>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_wgrad_kernel(const __grid_constant__ CUtensorMap mapDY,
                                                                  const __grid_constant__ CUtensorMap mapX, WgParams p) {
  constexpr int BOX = KP * 64 * 2;                  // one [KP pos][64 ch] box
  constexpr int A_BYTES = 2 * BOX, B_BYTES = (NT / 64) * BOX, STAGE_BYTES = A_BYTES + B_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int co0 = (blockIdx.x / p.ci_tiles) * 128, ci0 = (blockIdx.x % p.ci_tiles) * NT;
  const int tap = p.plain == 2 ? 0 : blockIdx.y, r = tap / 3, q = tap % 3;
  const int bz = p.plain == 2 ? blockIdx.y : 0;
  const int ks0 = blockIdx.z * p.per_split;
  const int ks1 = min(p.kstages, ks0 + p.per_split);
  const int KS = ks1 - ks0;
  if (warp == TC_CWARPS && lane == 0) {
    tma_prefetch_desc(&mapDY);
    tma_prefetch_desc(&mapX);
    for (int s = 0; s < STAGES; s++) { mbar_init(full_bar + s, 2); mbar_init(empty_bar + s, TC_CWARPS); }   // two producers
    fence_barrier_init();
  }
  __syncthreads();
  float acc[NT / 2];
  if (warp == TC_CWARPS) {
    if (lane == 0) {
      const int per_img = p.tiles_w * p.tiles_h;
      for (int i = 0; i < KS; i++) {
        const int s = i % STAGES;
        const uint32_t ph = (i / STAGES) & 1;
        mbar_wait(empty_bar + s, ph ^ 1);
        const int ks = ks0 + i;
        const int img = ks / per_img, rem = ks % per_img;
        const int h0 = (rem / p.tiles_w) * p.BH, w0 = (rem % p.tiles_w) * p.BW;
        uint8_t* sa = smem + s * STAGE_BYTES;
        mbar_expect_tx(full_bar + s, A_BYTES);
        if (p.plain == 2) {
          tma_load_3d(sa, &mapDY, full_bar + s, co0, ks * KP, bz);
          tma_load_3d(sa + BOX, &mapDY, full_bar + s, co0 + 64, ks * KP, bz);
        } else if (p.plain) {
          tma_load_2d(sa, &mapDY, full_bar + s, co0, ks * KP);
          tma_load_2d(sa + BOX, &mapDY, full_bar + s, co0 + 64, ks * KP);
        } else {
          tma_load_4d(sa, &mapDY, full_bar + s, co0, w0, h0, img);
          tma_load_4d(sa + BOX, &mapDY, full_bar + s, co0 + 64, w0, h0, img);
        }
      }
    }
    __syncwarp();
  } else if (warp == TC_CWARPS + 1) {
    if (lane == 0) {            // second producer: the X (B operand) boxes
      const int per_img = p.tiles_w * p.tiles_h;
      for (int i = 0; i < KS; i++) {
        const int s = i % STAGES;
        const uint32_t ph = (i / STAGES) & 1;
        mbar_wait(empty_bar + s, ph ^ 1);
        const int ks = ks0 + i;
        const int img = ks / per_img, rem = ks % per_img;
        const int h0 = (rem / p.tiles_w) * p.BH, w0 = (rem % p.tiles_w) * p.BW;
        uint8_t* sb = smem + s * STAGE_BYTES + A_BYTES;
        mbar_expect_tx(full_bar + s, B_BYTES);
        if (p.plain == 2) {
#pragma unroll
          for (int j = 0; j < NT / 64; j++) tma_load_3d(sb + j * BOX, &mapX, full_bar + s, ci0 + 64 * j, ks * KP, bz);
        } else if (p.plain) {
#pragma unroll
          for (int j = 0; j < NT / 64; j++) tma_load_2d(sb + j * BOX, &mapX, full_bar + s, ci0 + 64 * j, ks * KP);
        } else {
#pragma unroll
          for (int j = 0; j < NT / 64; j++)
            tma_load_4d(sb + j * BOX, &mapX, full_bar + s, ci0 + 64 * j, w0 + q - p.pad, h0 + r - p.pad, img);
        }
      }
    }
    __syncwarp();
  } else {
    // ===== consumers: warpgroup wg accumulates co rows [64 wg, 64 wg + 64) = A box wg =====
    const int wg = warp >> 2;
#pragma unroll
    for (int i = 0; i < NT / 2; i++) acc[i] = 0.f;
    for (int i = 0; i < KS; i++) {
      const int s = i % STAGES;
      const uint32_t ph = (i / STAGES) & 1;
      mbar_wait(full_bar + s, ph);
      const uint32_t sa = smem_u32(smem + s * STAGE_BYTES) + wg * BOX;
      const uint32_t sb = smem_u32(smem + s * STAGE_BYTES) + A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < KP / 16; k++)
        Wgmma<NT, 1, 1>::mma(acc, make_mnmajor_sw128_desc(sa + k * 2048, BOX), make_mnmajor_sw128_desc(sb + k * 2048, BOX), 1u);
      wgmma_commit();
      wgmma_wait0();
      wgmma_acc_fence<NT / 2>(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar + s);
    }
  }
  if (p.ordered && gridDim.z > 1) {
    // ordered split K: the splits of this tile are one cluster; rank 0 adds the partials in split order and alone writes dW
    float* part = reinterpret_cast<float*>(smem);      // the ring is idle once every consumer is past its last K block
    if (warp < TC_CWARPS) {
      asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
      for (int i = 0; i < NT / 2; i++) part[i * 256 + threadIdx.x] = acc[i];
    }
    cl_sync();
    if (cl_rank() == 0 && warp < TC_CWARPS) {
#pragma unroll
      for (int i = 0; i < NT / 2; i += 16) cl_sum_n<16>(part + i * 256 + threadIdx.x, 256, acc + i);
    }
    cl_sync();
    if (cl_rank() != 0) return;
  }
  if (warp < TC_CWARPS) {
    const int wg = warp >> 2, cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int co = co0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (co >= p.Cout) continue;
      float* orow = p.plain ? p.dw + (int64_t)bz * p.batch_c + (int64_t)co * p.ldc : p.dw + ((int64_t)co * 9 + tap) * p.Cin;
#pragma unroll
      for (int i = 0; i < NT / 8; i++) {                 // split-K partial sums (or, ordered, the tile's sum) onto C
        const int ci = ci0 + 8 * i + cq;
        if (ci < p.Cin) atomicAdd(orow + ci, acc[4 * i + 2 * h]);
        if (ci + 1 < p.Cin) atomicAdd(orow + ci + 1, acc[4 * i + 2 * h + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side: tensor maps + launch
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                        const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_tmapEncodeTiled g_encode = nullptr;
static int g_tc_state = -1;   // -1 unknown, 0 unavailable, 1 ok

bool tc_available() {
  if (g_tc_state >= 0) return g_tc_state == 1;
  g_tc_state = 0;
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess || major != 9) return false;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || fn == nullptr ||
      qres != cudaDriverEntryPointSuccess)
    return false;
  g_encode = (PFN_tmapEncodeTiled)fn;
  g_tc_state = 1;
  return true;
}

// cuTensorMapEncodeTiled costs ~1-2 us of host time; the decoder issues ~600 skinny GEMMs per step with a handful
// of distinct (pointer, shape) combinations per step index, so encoded maps are cached.
struct MapKey {
  const void* base; int rank; cuuint64_t dims[4]; cuuint64_t str[3]; cuuint32_t box[4];
  bool operator==(const MapKey& o) const { return memcmp(this, &o, sizeof(MapKey)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(MapKey) / 8; i++) { h ^= w[i]; h *= 1099511628211ull; }
    return (size_t)h;
  }
};
// the ABI allows one host thread per device: the descriptor cache is shared by all of them -> guarded
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;
static std::mutex g_map_mutex;

static int make_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                    const cuuint32_t* box) {
  MapKey key;
  memset(&key, 0, sizeof(key));
  key.base = base; key.rank = rank;
  for (int i = 0; i < rank; i++) { key.dims[i] = dims[i]; key.box[i] = box[i]; }
  for (int i = 0; i + 1 < rank; i++) key.str[i] = strides_bytes[i];
  {
    std::lock_guard<std::mutex> lk(g_map_mutex);
    auto it = g_map_cache.find(key);
    if (it != g_map_cache.end()) { *m = it->second; return LO_OK; }
  }
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(LO_ECUDA, "%s: cuTensorMapEncodeTiled failed (%ld)", "tc", (long)r);
  std::lock_guard<std::mutex> lk(g_map_mutex);
  if (g_map_cache.size() > 20000) g_map_cache.clear();
  g_map_cache.emplace(key, *m);
  return LO_OK;
}

long long* g_tc_dbg = nullptr;

template <int NT, int STAGES, int MC>
static int launch_tc(const CUtensorMap& mA, const CUtensorMap& mB, const TcParams& p, int mtiles, int splits, cudaStream_t st) {
  using SM = TcSmem<NT, STAGES>;
  static bool attr_set = false;
  if (!attr_set) {
    LO_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<NT, STAGES, MC>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::TOTAL));
    attr_set = true;
  }
  dim3 grid(cdiv(p.N, NT), mtiles, splits);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = SM::TOTAL;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (g_opt_pdl) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    n++;
  }
  if (MC) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = 2;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    n++;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  LO_CUDA(cudaLaunchKernelEx(&cfg, tc_gemm_kernel<NT, STAGES, MC>, mA, mB, p));
  LO_LAUNCH_OK();
  return LO_OK;
}

static int launch_tc_any(const CUtensorMap& mA, const CUtensorMap& mB, TcParams& p, int mtiles, int splits, int nt, cudaStream_t st,
                         int mc = 0) {
  const int KB = p.K / TC_BK;
  if (splits < 1) splits = 1;
  if (splits > KB) splits = KB;
  p.kb_per_split = cdiv(KB, splits);
  splits = cdiv(KB, p.kb_per_split);
  p.atomic = splits > 1 ? 1 : p.atomic;
  if (nt == 64 && mtiles == 1 && p.kb_per_split > 4 && g_opt_skinny8) return launch_tc<64, 8, 0>(mA, mB, p, mtiles, splits, st);   // skinny: all K in flight
  if (nt == 64) return launch_tc<64, 4, 0>(mA, mB, p, mtiles, splits, st);
  if (mc) return launch_tc<128, 3, 1>(mA, mB, p, mtiles, splits, st);
  return launch_tc<128, 3, 0>(mA, mB, p, mtiles, splits, st);
}

// splits > 1 (or atomic_acc): fp32 C only, partial sums are ADDED onto C with atomics (C must hold the base values)
int tc_gemm_nt_ex(const bf16* A, int64_t lda, const bf16* W, int64_t ldw, void* C, int dtC, int64_t ldc, int M, int N, int K,
                  const float* bias, int accumulate, int relu, int splits, int atomic_acc, int small_n_tile, cudaStream_t st) {
  if (!tc_available()) return fail(LO_ENOTSUP, "%s: needs an sm_90 device", __func__);
  LO_CHECK_ARG(K % 64 == 0 && lda % 8 == 0 && ldw % 8 == 0 && ldc % 8 == 0 && ldc >= (N + 7) / 8 * 8, "K%64, ld%8, ldc >= roundup8(N)");
  LO_CHECK_ARG(((uintptr_t)A & 15) == 0 && ((uintptr_t)W & 15) == 0 && ((uintptr_t)C & 15) == 0, "16-byte alignment");
  CUtensorMap mA, mB;
  const int NT = (N <= 64 || small_n_tile) ? 64 : 128;
  const int mc = (g_opt_conv_mc && NT == 128 && cdiv(N, 128) % 2 == 0 && splits <= 1 && !atomic_acc) ? 1 : 0;
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)M};
    cuuint64_t str[1] = {(cuuint64_t)lda * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)(mc ? 64 : 128)};
    LO_TRY(make_map(&mA, A, 2, dims, str, box));
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
    cuuint64_t str[1] = {(cuuint64_t)ldw * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)NT};
    LO_TRY(make_map(&mB, W, 2, dims, str, box));
  }
  LO_CHECK_ARG(!(splits > 1 || atomic_acc) || (dtC == LO_F32 && !relu), "split-K needs fp32 output without ReLU");
  TcParams p{};
  p.M = M; p.N = N; p.K = K;
  p.bias = bias; p.out = C; p.ldc = ldc;
  p.out_f32 = (dtC == LO_F32); p.accumulate = accumulate; p.relu = relu; p.atomic = atomic_acc;
  p.w_evict_last = (M <= 128) ? 1 : 0;
  p.dbg = g_tc_dbg;
  return launch_tc_any(mA, mB, p, cdiv(M, TC_BM), splits, NT, st, mc);
}

int tc_gemm_nt(const bf16* A, int64_t lda, const bf16* W, int64_t ldw, void* C, int dtC, int64_t ldc, int M, int N, int K,
               const float* bias, int accumulate, int relu, cudaStream_t st) {
  return tc_gemm_nt_ex(A, lda, W, ldw, C, dtC, ldc, M, N, K, bias, accumulate, relu, 1, 0, 0, st);
}

template <int NT, int STAGES, int MT>
static int launch_conv_p(const CUtensorMap& mA, const CUtensorMap& mB, const ConvParams& p, int mtiles, cudaStream_t st) {
  using SM = TcPSmem<NT, STAGES, MT>;
  static bool attr_set = false;
  static int n_sm = 0;
  if (!attr_set) {
    LO_CUDA(cudaFuncSetAttribute(tc_conv_p_kernel<NT, STAGES, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::TOTAL));
    int dev = 0;
    LO_CUDA(cudaGetDevice(&dev));
    LO_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    attr_set = true;
  }
  const int ntn = cdiv(p.N, NT);
  const int total = cdiv(mtiles, MT) * ntn;
  const int grid = total < n_sm ? total : n_sm;
  LO_CUDA(launch_pdl(tc_conv_p_kernel<NT, STAGES, MT>, dim3(grid), dim3(TC_THREADS), (size_t)SM::TOTAL, st, mA, mB, p, ntn, total, mtiles));
  LO_LAUNCH_OK();
  return LO_OK;
}

int tc_conv3x3(const bf16* x, const bf16* w, const float* bias, const bf16* mask, bf16* y, int N, int H, int W, int Cin, int Cout,
               int pad, int relu, cudaStream_t st) {
  if (!tc_available()) return fail(LO_ENOTSUP, "%s: needs an sm_90 device", __func__);
  LO_CHECK_ARG(Cin % 64 == 0 && Cout % 8 == 0, "Cin%64==0, Cout%8==0");
  const int Ho = H + 2 * pad - 2, Wo = W + 2 * pad - 2;
  int BW = 128;
  while (BW > 8 && BW / 2 >= Wo) BW /= 2;     // smallest power of two >= Wo (capped at 128)
  const int BH = 128 / BW;
  const int NT = Cout % 256 == 0 ? 256 : (Cout > 64 ? 128 : 64);
  CUtensorMap mA, mB;
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t str[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)W * Cin * 2, (cuuint64_t)H * W * Cin * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)BW, (cuuint32_t)BH, 1};
    LO_TRY(make_map(&mA, x, 4, dims, str, box));
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)9 * Cin, (cuuint64_t)Cout};
    cuuint64_t str[1] = {(cuuint64_t)9 * Cin * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)NT};
    LO_TRY(make_map(&mB, w, 2, dims, str, box));
  }
  ConvParams p{};
  p.N = Cout; p.K = 9 * Cin;
  p.Cin = Cin; p.pad = pad; p.Ho = Ho; p.Wo = Wo;
  p.BW = BW; p.BH = BH; p.tiles_w = cdiv(Wo, BW); p.tiles_h = cdiv(Ho, BH);
  p.bias = bias; p.mask = mask; p.out = y; p.ldc = Cout; p.relu = relu;
  const int mtiles = N * p.tiles_w * p.tiles_h;
  if (NT == 256) return launch_conv_p<256, 4, 1>(mA, mB, p, mtiles, st);
  if (NT == 128) return launch_conv_p<128, 4, 2>(mA, mB, p, mtiles, st);
  return launch_conv_p<64, 4, 2>(mA, mB, p, mtiles, st);
}


// K splits of a weight-gradient launch of `tiles` CTA tiles over `kstages` K blocks when `slots` CTAs are resident at once.
// The kernel holds one CTA per SM, so a short last wave takes about as long as a full one: the fewest CTAs whose last wave
// is at least 90 % full, every split keeping at least `min_ks` K blocks (a full ring); failing that, the fullest last wave.
static int whole_wave_splits(int tiles, int kstages, int min_ks, int slots) {
  int best = 1;
  double best_fill = -1.0;
  const int smax = kstages / min_ks > 1 ? kstages / min_ks : 1;
  for (int s = 1; s <= smax; s++) {
    const int splits = cdiv(kstages, cdiv(kstages, s));      // the count the rounded-up split length gives
    const long ctas = (long)tiles * splits;
    const double fill = (double)ctas / ((double)((ctas + slots - 1) / slots) * slots);
    if (fill >= 0.9) return splits;
    if (fill > best_fill) { best_fill = fill; best = splits; }
  }
  return best;
}

// One weight-gradient launch over a grid of (tiles_x, tiles_y) output tiles; p.kstages counts K blocks of KP positions.
// split_k: the K blocks are cut into splits along grid.z (whole waves, or with option "deterministic" the decomposition its
// ordered cluster sum was built on: two CTAs per SM targeted, at most 8 splits, counted for 128-channel tiles of 128-position
// blocks, so the split boundaries fall on the same positions for either tile shape).
template <int NT, int KP, int STAGES>
static int launch_wgrad(const CUtensorMap& mDY, const CUtensorMap& mX, WgParams& p, int tiles_x, int tiles_y, bool split_k,
                        cudaStream_t st) {
  constexpr int TOTAL = STAGES * (2 + NT / 64) * KP * 128 + 1024 + 256;
  static bool attr_set = false;
  if (!attr_set) {
    LO_CUDA(cudaFuncSetAttribute(tc_wgrad_kernel<NT, KP, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, TOTAL));
    attr_set = true;
  }
  const int tiles = tiles_x * tiles_y;
  if (!split_k) {
    p.per_split = p.kstages;
  } else if (g_opt_det) {
    constexpr int PB = 128 / KP;                                // K blocks per 128 positions
    const int ks128 = cdiv(p.kstages, PB);
    int s = cdiv(LO_NUM_SMS * 2, NT == 256 ? 2 * tiles : tiles);
    if (s > 8) s = 8;
    if (s > ks128) s = ks128;
    if (s < 1) s = 1;
    p.per_split = cdiv(ks128, s) * PB;
  } else {
    const int slots = resident_ctas((const void*)tc_wgrad_kernel<NT, KP, STAGES>, TC_THREADS, TOTAL);
    if (slots <= 0) return fail(LO_ECUDA, "%s: occupancy query failed", __func__);
    p.per_split = cdiv(p.kstages, whole_wave_splits(tiles, p.kstages, STAGES, slots));
  }
  const int splits = cdiv(p.kstages, p.per_split);
  p.ordered = g_opt_det && splits > 1;
  const dim3 grid(tiles_x, tiles_y, splits);
  if (p.ordered)
    LO_CUDA(launch_cluster(tc_wgrad_kernel<NT, KP, STAGES>, grid, dim3(TC_THREADS), (size_t)TOTAL, st, dim3(1, 1, splits), false, mDY, mX, p));
  else
    tc_wgrad_kernel<NT, KP, STAGES><<<grid, TC_THREADS, TOTAL, st>>>(mDY, mX, p);
  LO_LAUNCH_OK();
  return LO_OK;
}

// the weight gradient is ADDED onto dw (zero it for a plain product)
int tc_conv3x3_wgrad(const bf16* x, const bf16* dy, float* dw, int N, int H, int W, int Cin, int Cout, int pad, cudaStream_t st) {
  if (!tc_available()) return fail(LO_ENOTSUP, "%s: needs an sm_90 device", __func__);
  LO_CHECK_ARG(Cin % 64 == 0 && Cout % 128 == 0, "Cin%64==0, Cout%128==0");
  const int Ho = H + 2 * pad - 2, Wo = W + 2 * pad - 2;
  int BW = 128;
  while (BW > 8 && BW / 2 >= Wo) BW /= 2;
  const int BH = 128 / BW;
  // 128 (co) x 256 (ci) tiles when Cin allows it: 87 instead of 64 FLOP per byte pulled from L2, on 64-position K blocks
  const int NT = Cin % 256 == 0 ? 256 : (Cin >= 128 ? 128 : 64);
  WgParams p{};
  p.Cin = Cin; p.Cout = Cout; p.Ho = Ho; p.Wo = Wo; p.pad = pad;
  p.BW = BW; p.BH = BH; p.tiles_w = cdiv(Wo, BW); p.tiles_h = cdiv(Ho, BH);
  if (NT == 256) {
    // each 128-position box BW x BH becomes two 64-position boxes in the same row-major order: its upper and lower half
    // rows, or (one row of 128) its left and right half
    if (BH >= 2) { p.BH = BH / 2; p.tiles_h *= 2; }
    else { p.BW = BW / 2; p.tiles_w *= 2; }
  }
  p.kstages = N * p.tiles_w * p.tiles_h;
  p.dw = dw;
  p.ci_tiles = Cin / NT;
  CUtensorMap mDY, mX;
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cout, (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)N};
    cuuint64_t str[3] = {(cuuint64_t)Cout * 2, (cuuint64_t)Wo * Cout * 2, (cuuint64_t)Ho * Wo * Cout * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)p.BW, (cuuint32_t)p.BH, 1};
    LO_TRY(make_map(&mDY, dy, 4, dims, str, box));
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t str[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)W * Cin * 2, (cuuint64_t)H * W * Cin * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)p.BW, (cuuint32_t)p.BH, 1};
    LO_TRY(make_map(&mX, x, 4, dims, str, box));
  }
  const int tiles_x = (Cout / 128) * p.ci_tiles;
  if (NT == 256) return launch_wgrad<256, 64, 4>(mDY, mX, p, tiles_x, 9, true, st);
  if (NT == 128) return launch_wgrad<128, 128, 3>(mDY, mX, p, tiles_x, 9, true, st);
  return launch_wgrad<64, 128, 4>(mDY, mX, p, tiles_x, 9, true, st);
}

// C[M][N] (fp32, ldc) += A[K][M]^T * B[K][N]; A, B bf16 row-major.  C must hold the values to accumulate onto
// (zero it for a plain product): split-K partial sums land with fp32 atomics (in split order with option "deterministic").
int tc_gemm_tn(const bf16* A, int64_t lda, const bf16* B, int64_t ldb, float* C, int64_t ldc, int M, int N, int K, cudaStream_t st) {
  if (!tc_available()) return fail(LO_ENOTSUP, "%s: needs an sm_90 device", __func__);
  LO_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "lda%8, ldb%8");
  LO_CHECK_ARG(((uintptr_t)A & 15) == 0 && ((uintptr_t)B & 15) == 0, "16-byte alignment");
  // 128 x 128 tiles by default also where N % 256 == 0: with the decoder's K = B * T a split runs few K blocks, and the
  // 128 x 256 grid needs twice the splits (twice the fp32 atomics); measured slower on two of its four such GEMMs (DESIGN.md §8)
  const int NT = (g_opt_wgrad256 && N % 256 == 0) ? 256 : (N > 64 ? 128 : 64);
  const int KP = NT == 256 ? 64 : 128;                          // positions per K block
  CUtensorMap mA, mB;
  {
    cuuint64_t dims[2] = {(cuuint64_t)M, (cuuint64_t)K};
    cuuint64_t str[1] = {(cuuint64_t)lda * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)KP};
    LO_TRY(make_map(&mA, A, 2, dims, str, box));
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)N, (cuuint64_t)K};
    cuuint64_t str[1] = {(cuuint64_t)ldb * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)KP};
    LO_TRY(make_map(&mB, B, 2, dims, str, box));
  }
  WgParams p{};
  p.plain = 1; p.Cout = M; p.Cin = N; p.dw = C; p.ldc = ldc;
  p.tiles_w = p.tiles_h = 1; p.BW = KP; p.BH = 1;
  p.kstages = cdiv(K, KP);
  p.ci_tiles = cdiv(N, NT);
  const int tiles_x = cdiv(M, 128) * p.ci_tiles;
  if (NT == 256) return launch_wgrad<256, 64, 4>(mA, mB, p, tiles_x, 1, true, st);
  if (NT == 128) return launch_wgrad<128, 128, 3>(mA, mB, p, tiles_x, 1, true, st);
  return launch_wgrad<64, 128, 4>(mA, mB, p, tiles_x, 1, true, st);
}

// Batched C[b][M][N] (fp32) += A[b][K][M]^T * B[b][K][N]; A, B bf16 with arbitrary (16-byte multiple) strides:
// element (b, k, m) of A at A + b * sAb + k * sAk + m, likewise B.  One launch, grid.y = batch.  (decoder backward:
// d enc[b] += alphas[b]^T dctx[:, b, :], the context read summed over time.)
int tc_gemm_tn_batched(const bf16* A, int64_t sAk, int64_t sAb, const bf16* B, int64_t sBk, int64_t sBb, float* C, int64_t ldc,
                       int64_t sCb, int M, int N, int K, int batch, cudaStream_t st) {
  if (!tc_available()) return fail(LO_ENOTSUP, "%s: needs an sm_90 device", __func__);
  LO_CHECK_ARG(sAk % 8 == 0 && sAb % 8 == 0 && sBk % 8 == 0 && sBb % 8 == 0, "strides must be multiples of 8 elements");
  LO_CHECK_ARG(((uintptr_t)A & 15) == 0 && ((uintptr_t)B & 15) == 0 && batch >= 1 && batch <= 65535, "alignment / batch");
  CUtensorMap mA, mB;
  {
    cuuint64_t dims[3] = {(cuuint64_t)M, (cuuint64_t)K, (cuuint64_t)batch};
    cuuint64_t str[2] = {(cuuint64_t)sAk * 2, (cuuint64_t)sAb * 2};
    cuuint32_t box[3] = {64, 128, 1};
    LO_TRY(make_map(&mA, A, 3, dims, str, box));
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)N, (cuuint64_t)K, (cuuint64_t)batch};
    cuuint64_t str[2] = {(cuuint64_t)sBk * 2, (cuuint64_t)sBb * 2};
    cuuint32_t box[3] = {64, 128, 1};
    LO_TRY(make_map(&mB, B, 3, dims, str, box));
  }
  WgParams p{};
  p.plain = 2; p.Cout = M; p.Cin = N; p.dw = C; p.ldc = ldc; p.batch_c = sCb;
  p.tiles_w = p.tiles_h = 1; p.BW = 128; p.BH = 1;
  p.kstages = cdiv(K, 128);                     // no split-K: the batch dimension supplies the parallelism
  const int NT = N > 64 ? 128 : 64;
  p.ci_tiles = cdiv(N, NT);
  if (NT == 128) return launch_wgrad<128, 128, 3>(mA, mB, p, cdiv(M, 128) * p.ci_tiles, batch, false, st);
  return launch_wgrad<64, 128, 4>(mA, mB, p, cdiv(M, 128) * p.ci_tiles, batch, false, st);
}

}  // namespace lo
