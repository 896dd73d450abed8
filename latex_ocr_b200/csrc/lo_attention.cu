// Attention step kernels, version 2: the att1 / enc row streams go through a TMA bulk-copy (cp.async.bulk) ->
// shared-memory ring fed by a dedicated producer warp, so the bytes in flight per SM (2 CTAs x 3 stages x 32 KB)
// no longer depend on register-limited occupancy.  Same math, same combine order, same outputs as the register
// versions in lo_decoder.cu (attention_fwd_kernel / attention_bwd_kernel), which remain the fallback.
//   forward : e_r = w . relu(att1_r + att2) ; online softmax ; ctx = sum_r alpha_r enc_r      (seq2seq_torch.py:186-190)
//   backward: dalpha_r = <dctx, enc_r> + dreg_r ; de_r = alpha_r (dalpha_r - s) ; datt2 = w * sum_r de_r [att1_r + att2 > 0]
// L2 policy: att1 and enc do not change inside a time loop, so every step reads the same bytes in the same order, but a step
// streams twice the L2.  The forward pipe kernels and the tensor-core backward keep a fixed share of their ring stages in L2
// (att_keep_stage, att_keep_q: option att_l2_keep_mb) and stream the rest evict_first; the other backwards use fixed hints.
#include <cooperative_groups.h>

#include <mutex>
#include <vector>

#include "lo_common.cuh"
#include "lo_ptx.cuh"

namespace cg = cooperative_groups;

namespace lo {

#ifndef LO_ATT_RPW
#define LO_ATT_RPW 2          // rows per consumer warp per stage (bf16): 2 -> 32 KB stages, 2 CTAs/SM ; 1 -> 16 KB stages, 3 CTAs/SM
#endif
#ifndef LO_ATT_MINB
#define LO_ATT_MINB 2
#endif
#define AP_THREADS 288
#define AP_CWARPS 8
#define AP_STAGES 3
#define AP_MAXSPLIT 16


// ---- timing build only (-DLO_ATT_TIMING, tools/att_timeline.py): per-CTA %globaltimer stamps of the last attention launch
#ifdef LO_ATT_TIMING
__device__ long long* g_att_ts = nullptr;
__device__ __forceinline__ void att_ts(int k) {
  if (g_att_ts) {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    g_att_ts[((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * 16 + k] = t;
  }
}
#define ATT_TS(k, cond) do { if (cond) att_ts(k); } while (0)
#else
#define ATT_TS(k, cond) do { } while (0)
#endif

// L2 residency of ring stage i of a CTA.  The first `depth` stages are issued before griddepcontrol.wait, while the preceding
// small launches leave HBM idle, so an L2 hit gains nothing there: they always stream.  Of the later stages j = i - depth, a share
// keep_q / 1024 is kept, spread evenly (stage j is kept when floor((j + 1) q / 1024) > floor(j q / 1024)), so HBM stays busy
// while the hits are served.  The same stages are kept at every step of a time loop: the rule depends on nothing else.
// tests/test_l2_keep_rule.py mirrors it.
__host__ __device__ __forceinline__ bool att_keep_stage(int i, int depth, int keep_q) {
  const int j = i - depth;
  return j >= 0 && (((j + 1) * keep_q) >> 10) != ((j * keep_q) >> 10);
}

// score non-linearity: ACT 0 = ReLU (torch flavour, seq2seq_torch.py:188), 1 = tanh (Genthial cell, attention_mechanism.py:82)
template <int ACT, bool APPROX>
__device__ __forceinline__ float att_act(float x) {
  if constexpr (ACT == 0) return fmaxf(x, 0.f);
  else if constexpr (APPROX) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
  } else return tanhf(x);
}
// derivative given the pre-activation (ReLU) / the activation value (tanh)
template <int ACT>
__device__ __forceinline__ float att_dact(float pre, float post) {
  if constexpr (ACT == 0) return pre > 0.f ? 1.f : 0.f;
  else return 1.f - post * post;
}

// rows per split of the BACKWARD mask kernels: even, so that every stage starts on an (even, odd) row pair of the mask layout
__host__ __device__ __forceinline__ int att_rows_per_split(int R, int nsplit) { return (((R + nsplit - 1) / nsplit) + 1) & ~1; }

// NVA / NVC: 256-element groups per att1 row / per enc row (the torch flavour has A = C; the Genthial cell dim_e = 256 < C = 512)
template <typename T, int NVA, int NVC>
struct ApCfg {
  static constexpr int CHA = NVA * 256;
  static constexpr int CHC = NVC * 256;
  static constexpr int NVM = NVA > NVC ? NVA : NVC;
  static constexpr int RPW = (sizeof(T) == 2 && NVM <= 2) ? LO_ATT_RPW : 1;      // rows per consumer warp per stage
  static constexpr int ROWS = AP_CWARPS * RPW;
  static constexpr int HALF_A = ROWS * CHA;                             // att1 part
  static constexpr int HALF_C = ROWS * CHC;                             // enc part
  static constexpr int STAGE_ELEMS = HALF_A + HALF_C;
  static constexpr int STAGE_BYTES = STAGE_ELEMS * (int)sizeof(T);
  static constexpr int SMEM = AP_STAGES * STAGE_BYTES + 128;
};

// The work of one CTA: split sp of the nsplit splits of batch row b, which attends over the R regions of its image, rows g0.. of
// att1 / enc.  The CTA streams regions [sp * ceil(R / nsplit), ...) and, cluster-free, writes its partial sums to split slot
// pbase + sp of `partials` (pbase: the row's first slot) and takes a ticket at counters[b].  Called by the dense kernel (every row has
// R regions and nsplit splits) and by the ragged one (per-row R and nsplit from its CTA map).
template <typename T, int NVA, int NVC, bool CL, int ACT, bool MK>
__device__ __forceinline__ void attention_fwd_pipe_cta(
    const T* __restrict__ att1, const T* __restrict__ enc, const float* __restrict__ att2, int64_t att2_stride,
    const float* __restrict__ wf, float* __restrict__ alpha, int64_t alpha_stride, float* __restrict__ ctx,
    float* __restrict__ gate_pre, int64_t gate_stride, float* __restrict__ gctx, bf16* __restrict__ gctx_bf, int R, int nsplit,
    int* __restrict__ counters, float* __restrict__ partials, int keep_q, uint8_t* __restrict__ mask_out, int b, int sp, int64_t g0,
    int64_t pbase) {
  using C = ApCfg<T, NVA, NVC>;
  constexpr int CHA = C::CHA, CHC = C::CHC;
  extern __shared__ __align__(128) uint8_t ap_smem[];
  T* ring = reinterpret_cast<T*>(ap_smem);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ap_smem + AP_STAGES * C::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + AP_STAGES;
  float* s_e = reinterpret_cast<float*>(ap_smem + AP_STAGES * C::STAGE_BYTES + 128);   // cluster mode: raw scores of this CTA's rows
  __shared__ float s_m[AP_CWARPS], s_l[AP_CWARPS];
  __shared__ float s_msplit[AP_MAXSPLIT], s_lsplit[AP_MAXSPLIT];     // cluster-free combine: (M, L) of every split
  __shared__ int s_last;

  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int rps = (R + nsplit - 1) / nsplit;
  const int r0 = sp * rps, r1 = min(R, r0 + rps);
  const int nst = r1 > r0 ? (r1 - r0 + C::ROWS - 1) / C::ROWS : 0;
  const T* a1b = att1 + g0 * CHA;
  const T* eb = enc + g0 * CHC;
  float* alb = alpha + (int64_t)b * alpha_stride;
  ATT_TS(0, threadIdx.x == 0);

  if (threadIdx.x == 0) {
    for (int s = 0; s < AP_STAGES; s++) {
      mbar_init(full_bar + s, 1);
      mbar_init(empty_bar + s, AP_CWARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  // PDL: the producer's bulk copies read only loop-invariant tensors (att1, enc: written long before the preceding kernel), so they
  // are issued BEFORE griddepcontrol.wait and overlap the tail of the preceding launch; consumers wait before touching its results.
  float m = -INFINITY, l = 0.f;
  float gate_pf = 0.f;
  float acc[NVC * 8];
#pragma unroll
  for (int i = 0; i < NVC * 8; i++) acc[i] = 0.f;

  if (wid == AP_CWARPS) {
    // ===== producer warp: one lane issues the bulk copies =====
    if (lane == 0) {
      const uint64_t pk = l2_policy_evict_normal(), ps = l2_policy_evict_first();
      for (int i = 0; i < nst; i++) {
        const int s = i % AP_STAGES;
        const uint32_t ph = (i / AP_STAGES) & 1;
        mbar_wait(empty_bar + s, ph ^ 1);
        const int row = r0 + i * C::ROWS;
        const int rows = min(C::ROWS, r1 - row);
        const uint32_t bytes_a = (uint32_t)rows * CHA * (uint32_t)sizeof(T), bytes_c = (uint32_t)rows * CHC * (uint32_t)sizeof(T);
        T* sa = ring + (size_t)s * C::STAGE_ELEMS;
        const uint64_t pol = att_keep_stage(i, AP_STAGES, keep_q) ? pk : ps;      // att1 and enc rows of a stage stay together
        mbar_expect_tx(full_bar + s, bytes_a + bytes_c);
        ATT_TS(6, i == 0);
        ATT_TS(7, i == nst - 1);
        bulk_g2s(sa, a1b + (int64_t)row * CHA, bytes_a, full_bar + s, pol);
        bulk_g2s(sa + C::HALF_A, eb + (int64_t)row * CHC, bytes_c, full_bar + s, pol);
      }
    }
    __syncwarp();
    pdl_wait();          // the producer warp joins the combine below, which reads the preceding kernel's results
  } else {
    // ===== consumer warps =====
    float a2[NVA * 8], wv[NVA * 8];
#pragma unroll
    for (int j = 0; j < NVA; j++) ld8(wf + (j * 32 + lane) * 8, wv + j * 8);        // a parameter: independent of the preceding launch
    pdl_wait();
    ATT_TS(1, threadIdx.x == 0);
    pdl_trigger();
#pragma unroll
    for (int j = 0; j < NVA; j++) ld8(att2 + (int64_t)b * att2_stride + (j * 32 + lane) * 8, a2 + j * 8);
    // cluster mode: the gate pre-activation of the channel this thread finalises after the combine (one L2 round trip off the tail)
    if (CL && gate_pre && (int)threadIdx.x < (CHC + nsplit - 1) / nsplit && sp * ((CHC + nsplit - 1) / nsplit) + (int)threadIdx.x < CHC)
      gate_pf = gate_pre[(int64_t)b * gate_stride + sp * ((CHC + nsplit - 1) / nsplit) + threadIdx.x];
    ATT_TS(2, threadIdx.x == 0);
    for (int i = 0; i < nst; i++) {
      const int s = i % AP_STAGES;
      const uint32_t ph = (i / AP_STAGES) & 1;
      const int row = r0 + i * C::ROWS;
      const int rows = min(C::ROWS, r1 - row);
      mbar_wait(full_bar + s, ph);
      ATT_TS(3, threadIdx.x == 0 && i == 0);
      const uint32_t sa = smem_u32(ring + (size_t)s * C::STAGE_ELEMS);
      const uint32_t se = sa + C::HALF_A * (uint32_t)sizeof(T);
      constexpr uint32_t ES = (uint32_t)sizeof(T);
      const int ra = wid, rb = wid + AP_CWARPS;
      const bool one = ra < rows;
      const bool two = (C::RPW == 2) && (rb < rows);
      if (one) {
        float e0 = 0.f, e1 = 0.f;
        // training (ReLU score): bit 7 - (c % 8) of byte c/8 of row r = (att1[r][c] + att2[c] > 0); the backward reads these
        // 64 bytes per row instead of the 1 KB att1 row
        // layout: byte (r, c/8) at (r/2) * 2*(CHA/8) + (c/8)*2 + (r&1) — the bytes of an (even, odd) row pair are adjacent, which
        // is what the tensor-core backward wants (one 32-bit word per lane = its four A fragments of a 16 x 16 block)
        uint8_t* mrow = MK ? mask_out + (int64_t)b * ((R + 1) & ~1) * (CHA / 8) : nullptr;
#pragma unroll
        for (int j = 0; j < NVA; j++) {
          float v[8];
          lds8(sa + ((uint32_t)ra * CHA + (j * 32 + lane) * 8) * ES, v, (const T*)nullptr);
          uint32_t bits = 0;
#pragma unroll
          for (int q = 0; q < 8; q++) {
            const float pre = v[q] + a2[j * 8 + q];
            // one funnel shift per element collects the SIGN bits (element q -> bit 7-q); pre > 0 <=> sign clear, except for
            // pre == +0 exactly, where the ReLU subgradient is a convention and which a sum of a bf16 and an fp32 never hits
            if (MK) bits = __funnelshift_l(__float_as_uint(pre), bits, 1);
            e0 = fmaf(wv[j * 8 + q], att_act<ACT, sizeof(T) == 2>(pre), e0);
          }
          if (MK) mrow[(int64_t)((row + ra) >> 1) * (CHA / 4) + (j * 32 + lane) * 2 + ((row + ra) & 1)] = (uint8_t)(~bits);
          if (two) {
            lds8(sa + ((uint32_t)rb * CHA + (j * 32 + lane) * 8) * ES, v, (const T*)nullptr);
            bits = 0;
#pragma unroll
            for (int q = 0; q < 8; q++) {
              const float pre = v[q] + a2[j * 8 + q];
              if (MK) bits = __funnelshift_l(__float_as_uint(pre), bits, 1);
              e1 = fmaf(wv[j * 8 + q], att_act<ACT, sizeof(T) == 2>(pre), e1);
            }
            if (MK) mrow[(int64_t)((row + rb) >> 1) * (CHA / 4) + (j * 32 + lane) * 2 + ((row + rb) & 1)] = (uint8_t)(~bits);
          }
        }
        e0 = warp_sum(e0);
        e1 = warp_sum(e1);
        if (lane == 0) {
          if constexpr (CL) {
            s_e[row + ra - r0] = e0;
            if (two) s_e[row + rb - r0] = e1;
          } else {
            alb[row + ra] = e0;
            if (two) alb[row + rb] = e1;
          }
        }
        const float mn = two ? fmaxf(m, fmaxf(e0, e1)) : fmaxf(m, e0);
        const float sc = expf(m - mn);
        const float p0 = expf(e0 - mn);
        const float p1 = two ? expf(e1 - mn) : 0.f;
        l = l * sc + p0 + p1;
#pragma unroll
        for (int j = 0; j < NVC; j++) {
          float u[8];
          lds8(se + ((uint32_t)ra * CHC + (j * 32 + lane) * 8) * ES, u, (const T*)nullptr);
#pragma unroll
          for (int q = 0; q < 8; q++) acc[j * 8 + q] = fmaf(p0, u[q], acc[j * 8 + q] * sc);
          if (two) {
            lds8(se + ((uint32_t)rb * CHC + (j * 32 + lane) * 8) * ES, u, (const T*)nullptr);
#pragma unroll
            for (int q = 0; q < 8; q++) acc[j * 8 + q] = fmaf(p1, u[q], acc[j * 8 + q]);
          }
        }
        m = mn;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar + s);
    }
  }
  ATT_TS(4, threadIdx.x == 0);
  // cluster-free: the gate pre-activations of the channels this thread finalises should its CTA combine last (channel c = tid +
  // k * AP_THREADS, below).  Fetched here, so that the load hides behind the CTA combine and the ticket instead of sitting on the
  // last CTA's tail; only that CTA uses them.  Nothing else writes gate_pre before that CTA's ticket.
  constexpr int NCI = (CHC + AP_THREADS - 1) / AP_THREADS;
  float gpf[NCI];
  if constexpr (!CL) {
#pragma unroll
    for (int k = 0; k < NCI; k++) {
      const int c = threadIdx.x + k * AP_THREADS;
      gpf[k] = (gate_pre && c < CHC) ? gate_pre[(int64_t)b * gate_stride + c] : 0.f;
    }
  }
  __syncthreads();     // every TMA write has landed and been consumed: the ring can be reused for the combine
  ATT_TS(8, threadIdx.x == 0);
  float* s_acc = reinterpret_cast<float*>(ap_smem);          // [AP_CWARPS][CHC]
  if (wid < AP_CWARPS) {
    if (lane == 0) { s_m[wid] = m; s_l[wid] = l; }
#pragma unroll
    for (int j = 0; j < NVC; j++)
#pragma unroll
      for (int i = 0; i < 8; i++) s_acc[wid * CHC + (j * 32 + lane) * 8 + i] = acc[j * 8 + i];
  }
  __syncthreads();
  float M = -INFINITY;
#pragma unroll
  for (int w = 0; w < AP_CWARPS; w++) M = fmaxf(M, s_m[w]);
  float L = 0.f;
  float wsc[AP_CWARPS];
#pragma unroll
  for (int w = 0; w < AP_CWARPS; w++) {
    wsc[w] = (s_m[w] == -INFINITY) ? 0.f : expf(s_m[w] - M);
    L += s_l[w] * wsc[w];
  }
  if constexpr (CL) {
    // ===== cluster combine: the nsplit CTAs of this batch row exchange (M, L, acc) through distributed shared memory =====
    cg::cluster_group cluster = cg::this_cluster();
    float* s_part = s_acc + AP_CWARPS * CHC;                 // [CHC] combined accumulator of this CTA (still inside the ring)
    __shared__ float s_MLp[2];
    for (int c = threadIdx.x; c < CHC; c += AP_THREADS) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < AP_CWARPS; w++) t = fmaf(s_acc[w * CHC + c], wsc[w], t);
      s_part[c] = t;
    }
    if (threadIdx.x == 0) { s_MLp[0] = M; s_MLp[1] = L; }
    cluster.sync();
    float Mg = -INFINITY;
    for (int q = 0; q < nsplit; q++) Mg = fmaxf(Mg, cluster.map_shared_rank(s_MLp, q)[0]);
    float Lg = 0.f;
    float scl[8];
#pragma unroll
    for (int q = 0; q < 8; q++) {
      scl[q] = 0.f;
      if (q < nsplit) {
        const float* ml = cluster.map_shared_rank(s_MLp, q);
        const float ms = ml[0];
        scl[q] = (ms == -INFINITY) ? 0.f : expf(ms - Mg);
        Lg += ml[1] * scl[q];
      }
    }
    const float invL = 1.0f / Lg;
    // this CTA finalises its slice of the channels ...
    const int cps = (CHC + nsplit - 1) / nsplit;
    for (int c = sp * cps + threadIdx.x; c < min(CHC, (sp + 1) * cps); c += AP_THREADS) {
      float t = 0.f;
#pragma unroll
      for (int q = 0; q < 8; q++)
        if (q < nsplit) t = fmaf(cluster.map_shared_rank(s_part, q)[c], scl[q], t);
      t *= invL;
      ctx[(int64_t)b * CHC + c] = t;
      if (gate_pre) {
        const bool pf = c == sp * cps + (int)threadIdx.x && (int)threadIdx.x < AP_CWARPS * 32;     // fetched before the main loop
        const float g = sigmoidf_(pf ? gate_pf : gate_pre[(int64_t)b * gate_stride + c]);
        gate_pre[(int64_t)b * gate_stride + c] = g;
        gctx[(int64_t)b * CHC + c] = g * t;
        if (gctx_bf) gctx_bf[(int64_t)b * CHC + c] = __float2bfloat16_rn(g * t);
      } else if (gctx_bf) {
        gctx_bf[(int64_t)b * CHC + c] = __float2bfloat16_rn(t);      // no gate (Genthial cell): bf16 mirror of the context itself
      }
    }
    // ... and normalises the attention weights of its own rows (scores never leave shared memory)
    for (int r = r0 + threadIdx.x; r < r1; r += AP_THREADS) alb[r] = expf(s_e[r - r0] - Mg) * invL;
    cluster.sync();                                          // peers may still be reading this CTA's shared memory
    ATT_TS(5, threadIdx.x == 0);
    return;
  }
  float* part = partials + (pbase + sp) * (CHC + 2);
  for (int c = threadIdx.x; c < CHC; c += AP_THREADS) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < AP_CWARPS; w++) t = fmaf(s_acc[w * CHC + c], wsc[w], t);
    part[2 + c] = t;
  }
  if (threadIdx.x == 0) { part[0] = M; part[1] = L; }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int ticket = atomicAdd(counters + b, 1);
    s_last = (ticket == nsplit - 1);
    if (s_last) counters[b] = 0;
  }
  __syncthreads();
  if (!s_last) {
    ATT_TS(5, threadIdx.x == 0);
    return;
  }
  __threadfence();
  ATT_TS(9, threadIdx.x == 0);
  // ===== ordered combine by the CTA that took the last ticket: the same operations in the same split order as the cluster combine.
  // Every load it needs is issued before the first use: the splits' (M, L) into shared memory, this thread's partial sums of its
  // first channel and its first raw scores into registers, so the tail costs about one L2 round trip instead of a chain of them.
  const float* pb = partials + pbase * (CHC + 2);
  constexpr int PS = 8;      // partial sums of a channel held in registers; splits beyond PS are read in the loop
  constexpr int RB = 4;      // raw scores per thread held in registers; rows beyond RB * AP_THREADS are read in the loop
  if ((int)threadIdx.x < nsplit) {
    s_msplit[threadIdx.x] = __ldcg(pb + (int64_t)threadIdx.x * (CHC + 2));          // M of split tid
    s_lsplit[threadIdx.x] = __ldcg(pb + (int64_t)threadIdx.x * (CHC + 2) + 1);       // L of split tid
  }
  float pv[PS], ev[RB];
  auto load_parts = [&](int c) {
#pragma unroll
    for (int s = 0; s < PS; s++) pv[s] = s < nsplit ? __ldcg(pb + (int64_t)s * (CHC + 2) + 2 + c) : 0.f;
  };
  if ((int)threadIdx.x < CHC) load_parts(threadIdx.x);
#pragma unroll
  for (int k = 0; k < RB; k++) {
    const int r = threadIdx.x + k * AP_THREADS;
    ev[k] = r < R ? __ldcg(alb + r) : 0.f;
  }
  __syncthreads();
  float Mg = -INFINITY;
  for (int s = 0; s < nsplit; s++) Mg = fmaxf(Mg, s_msplit[s]);
  auto split_scale = [&](int s) {
    const float ms = s_msplit[s];
    return (ms == -INFINITY) ? 0.f : expf(ms - Mg);
  };
  float Lg = 0.f;
  for (int s = 0; s < nsplit; s++) Lg += s_lsplit[s] * split_scale(s);
  const float invL = 1.0f / Lg;
#pragma unroll
  for (int k = 0; k < NCI; k++) {
    const int c = threadIdx.x + k * AP_THREADS;
    if (c < CHC) {
      if (k > 0) load_parts(c);
      float t = 0.f;
#pragma unroll
      for (int s = 0; s < PS; s++)
        if (s < nsplit) t = fmaf(pv[s], split_scale(s), t);
      for (int s = PS; s < nsplit; s++) t = fmaf(__ldcg(pb + (int64_t)s * (CHC + 2) + 2 + c), split_scale(s), t);
      t *= invL;
      ctx[(int64_t)b * CHC + c] = t;
      if (gate_pre) {
        const float g = sigmoidf_(gpf[k]);
        gate_pre[(int64_t)b * gate_stride + c] = g;
        gctx[(int64_t)b * CHC + c] = g * t;
        if (gctx_bf) gctx_bf[(int64_t)b * CHC + c] = __float2bfloat16_rn(g * t);
      } else if (gctx_bf) {
        gctx_bf[(int64_t)b * CHC + c] = __float2bfloat16_rn(t);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < RB; k++) {
    const int r = threadIdx.x + k * AP_THREADS;
    if (r < R) alb[r] = expf(ev[k] - Mg) * invL;
  }
  for (int r = threadIdx.x + RB * AP_THREADS; r < R; r += AP_THREADS) alb[r] = expf(__ldcg(alb + r) - Mg) * invL;
  ATT_TS(5, threadIdx.x == 0);
}

// Dense layout: grid (nsplit, B), every image R regions, att1 / enc [B / rpi][R][.].
template <typename T, int NVA, int NVC, bool CL, int ACT, bool MK>
__global__ void __launch_bounds__(AP_THREADS, LO_ATT_MINB) attention_fwd_pipe_kernel(
    const T* __restrict__ att1, const T* __restrict__ enc, const float* __restrict__ att2, int64_t att2_stride,
    const float* __restrict__ wf, float* __restrict__ alpha, int64_t alpha_stride, float* __restrict__ ctx,
    float* __restrict__ gate_pre, int64_t gate_stride, float* __restrict__ gctx, bf16* __restrict__ gctx_bf, int R, int nsplit,
    int* __restrict__ counters, float* __restrict__ partials, int keep_q, int rpi, uint8_t* __restrict__ mask_out) {
  const int b = blockIdx.y, sp = blockIdx.x;
  // beam search: rpi consecutive rows attend over one image
  attention_fwd_pipe_cta<T, NVA, NVC, CL, ACT, MK>(att1, enc, att2, att2_stride, wf, alpha, alpha_stride, ctx, gate_pre, gate_stride, gctx,
                                                  gctx_bf, R, nsplit, counters, partials, keep_q, mask_out, b, sp,
                                                  (int64_t)(b / rpi) * R, (int64_t)b * nsplit);
}

// Ragged layout (decode of images of different sizes): image i owns regions [reg_off[i], reg_off[i+1]) of the packed att1 / enc.
// One-dimensional cluster-free grid; CTA x does the work cta_map[x] = {row b, split, splits of row b, first partial slot of row b}
// says (attention_ragged_map_kernel).  Decode only, no mask bits: ReLU score (ACT = 0, torch flavour) or tanh (ACT = 1, Genthial cell).
template <typename T, int NVA, int NVC, int ACT>
__global__ void __launch_bounds__(AP_THREADS, LO_ATT_MINB) attention_fwd_ragged_kernel(
    const T* __restrict__ att1, const T* __restrict__ enc, const float* __restrict__ att2, int64_t att2_stride,
    const float* __restrict__ wf, float* __restrict__ alpha, int64_t alpha_stride, float* __restrict__ ctx,
    float* __restrict__ gate_pre, int64_t gate_stride, float* __restrict__ gctx, bf16* __restrict__ gctx_bf,
    const int4* __restrict__ cta_map, const int32_t* __restrict__ reg_off, int rpi, int* __restrict__ counters,
    float* __restrict__ partials, int keep_q) {
  // the map and the offsets were written by the decode call's prologue, long before the preceding launch: read before its wait
  const int4 e = cta_map[blockIdx.x];
  const int img = e.x / rpi;
  const int g0 = reg_off[img];
  attention_fwd_pipe_cta<T, NVA, NVC, false, ACT, false>(att1, enc, att2, att2_stride, wf, alpha, alpha_stride, ctx, gate_pre, gate_stride,
                                                        gctx, gctx_bf, reg_off[img + 1] - g0, e.z, counters, partials, keep_q, nullptr,
                                                        e.x, e.y, (int64_t)g0, (int64_t)e.w);
}

// Splits of one row of the ragged launch: its share of ns * B splits in proportion to its region count, at least 1 and at most
// AP_MAXSPLIT; `fixed` (the att_nsplit option) gives every row ns.  Equal counts give every row exactly ns, the dense partition.
__host__ __device__ __forceinline__ int att_ragged_row_splits(int ns, int B, int Ri, int64_t sumR, bool fixed) {
  if (fixed) return ns;
  const int64_t q = (int64_t)ns * B * Ri / sumR;
  return q < 1 ? 1 : (q > AP_MAXSPLIT ? AP_MAXSPLIT : (int)q);
}

// One block: cta_map of the ragged launch (row-major: the splits of row 0, then row 1, ...) and zeroed ticket counters.
__global__ void attention_ragged_map_kernel(const int32_t* __restrict__ reg_off, int B, int rpi, int ns, int64_t sumR, int fixed,
                                            int4* __restrict__ cta_map, int* __restrict__ counters) {
  extern __shared__ int s_rows[];          // [B] splits of each row, then [B] first slot of each row
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    s_rows[b] = att_ragged_row_splits(ns, B, reg_off[b / rpi + 1] - reg_off[b / rpi], sumR, fixed != 0);
    counters[b] = 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int p = 0;
    for (int b = 0; b < B; b++) {
      s_rows[B + b] = p;
      p += s_rows[b];
    }
  }
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x)
    for (int s = 0; s < s_rows[b]; s++) cta_map[s_rows[B + b] + s] = make_int4(b, s, s_rows[b], s_rows[B + b]);
}

// DA1 (lo_attention_step_backward, a single Attention.forward call): while a stage is resident the consumer warps also store
//   datt1[b][r][a] = wf[a] * de[b][r] * act'(att1[b][r][a] + att2[b][a])
// in the storage type, so the att1 rows are read once for de, datt2, the d w_full partial and d att1.  Without DA1 the datt1
// argument (last, so the other parameters keep their offsets) is unused.
template <typename T, int NVA, int NVC, bool CL, int ACT, bool DA1 = false>
__global__ void __launch_bounds__(AP_THREADS) attention_bwd_pipe_kernel(
    const T* __restrict__ att1, const T* __restrict__ enc, const float* __restrict__ att2, const float* __restrict__ gate,
    int64_t o1_stride, const float* __restrict__ wf, const float* __restrict__ alpha, int64_t alpha_stride,
    const float* __restrict__ ctx, const float* __restrict__ dgctx, int64_t dg_stride, const float* __restrict__ dreg,
    int64_t dreg_stride, const float* __restrict__ sreg, int64_t sreg_stride, float* __restrict__ de, float* __restrict__ datt2,
    float* __restrict__ dgp, int64_t dcat_stride, bf16* __restrict__ datt2_bf, bf16* __restrict__ dgp_bf,
    float* __restrict__ dctx_out, int R, int nsplit, int* __restrict__ counters, float* __restrict__ partials,
    float* __restrict__ dwf_part, T* __restrict__ datt1) {
  using C = ApCfg<T, NVA, NVC>;
  constexpr int CHA = C::CHA, CHC = C::CHC;
  extern __shared__ __align__(128) uint8_t ap_smem[];
  T* ring = reinterpret_cast<T*>(ap_smem);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ap_smem + AP_STAGES * C::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + AP_STAGES;
  __shared__ int s_last;
  const int b = blockIdx.y, sp = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int rps = (R + nsplit - 1) / nsplit;
  const int r0 = sp * rps, r1 = min(R, r0 + rps);
  const int nst = r1 > r0 ? (r1 - r0 + C::ROWS - 1) / C::ROWS : 0;
  const T* a1b = att1 + (int64_t)b * R * CHA;
  const T* eb = enc + (int64_t)b * R * CHC;
  const float* s_wf = nullptr;           // DA1, NVA > 2: full_att.weight in shared memory (in registers it would spill)
  if constexpr (DA1 && NVA > 2) {
    __shared__ __align__(16) float s_wbuf[CHA];       // read 8 floats at a time (two 16-byte loads)
    for (int c = threadIdx.x; c < CHA; c += AP_THREADS) s_wbuf[c] = wf[c];
    s_wf = s_wbuf;
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < AP_STAGES; s++) {
      mbar_init(full_bar + s, 1);
      mbar_init(empty_bar + s, AP_CWARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  // PDL: the producer's bulk copies read only loop-invariant tensors (att1, enc: written long before the preceding kernel), so they
  // are issued BEFORE griddepcontrol.wait and overlap the tail of the preceding launch; consumers wait before touching its results.
  float macc[NVA * 8], wacc[NVA * 8];     // wacc: d w_full partial = sum_r de_r * relu(att1_r + att2)   (full_att.weight gradient)
#pragma unroll
  for (int i = 0; i < NVA * 8; i++) { macc[i] = 0.f; wacc[i] = 0.f; }

  if (wid == AP_CWARPS) {
    if (lane == 0) {
      const uint64_t pe = l2_policy_evict_last(), pa = l2_policy_evict_first();
      for (int i = 0; i < nst; i++) {
        const int s = i % AP_STAGES;
        const uint32_t ph = (i / AP_STAGES) & 1;
        mbar_wait(empty_bar + s, ph ^ 1);
        const int row = r0 + i * C::ROWS;
        const int rows = min(C::ROWS, r1 - row);
        const uint32_t bytes_a = (uint32_t)rows * CHA * (uint32_t)sizeof(T), bytes_c = (uint32_t)rows * CHC * (uint32_t)sizeof(T);
        T* sa = ring + (size_t)s * C::STAGE_ELEMS;
        mbar_expect_tx(full_bar + s, bytes_a + bytes_c);
        bulk_g2s(sa, a1b + (int64_t)row * CHA, bytes_a, full_bar + s, pa);
        bulk_g2s(sa + C::HALF_A, eb + (int64_t)row * CHC, bytes_c, full_bar + s, pe);
      }
    }
    __syncwarp();
    pdl_wait();          // the producer warp joins the combine below, which reads the preceding kernel's results
  } else {
    float a2[NVA * 8], dc[NVC * 8];
    float wv[NVA * 8];                 // DA1, NVA <= 2: full_att.weight in registers
    if constexpr (DA1 && NVA <= 2) {
#pragma unroll
      for (int j = 0; j < NVA; j++) ld8(wf + (j * 32 + lane) * 8, wv + j * 8);
    }
    float sdot = 0.f;
    // att2 / gate / ctx / sreg were saved by the forward pass: they are fetched BEFORE griddepcontrol.wait (overlapping the tail of
    // the preceding launch); only d gctx comes from the preceding kernel
    float gv[NVC * 8], cxv[NVC * 8];
#pragma unroll
    for (int j = 0; j < NVA; j++) ld8(att2 + (int64_t)b * o1_stride + (j * 32 + lane) * 8, a2 + j * 8);
#pragma unroll
    for (int j = 0; j < NVC; j++) {
      const int c0 = (j * 32 + lane) * 8;
      if (gate) ld8(gate + (int64_t)b * o1_stride + c0, gv + j * 8);
      ld8(ctx + (int64_t)b * CHC + c0, cxv + j * 8);
    }
    const float sreg_b = sreg ? sreg[(int64_t)b * sreg_stride] : 0.f;
    pdl_wait();
    pdl_trigger();
#pragma unroll
    for (int j = 0; j < NVC; j++) {
      const int c0 = (j * 32 + lane) * 8;
      float dg[8], gp[8];
      const float* g = gv + j * 8;
      const float* cx = cxv + j * 8;
      ld8(dgctx + (int64_t)b * dg_stride + c0, dg);
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const float gi = gate ? g[i] : 1.f;                // Genthial cell: the context is used ungated
        dc[j * 8 + i] = dg[i] * gi;
        sdot = fmaf(dc[j * 8 + i], cx[i], sdot);
        gp[i] = dg[i] * cx[i] * gi * (1.f - gi);
      }
      if (sp == 0 && wid == 0) {
        if (dgp) st8(dgp + (int64_t)b * dcat_stride + c0, gp);
        if (dgp_bf) st8(dgp_bf + (int64_t)b * dcat_stride + c0, gp);
        if (dctx_out) st8(dctx_out + (int64_t)b * CHC + c0, dc + j * 8);
      }
    }
    const float sall = warp_sum(sdot) + sreg_b;
    const float* alb = alpha + (int64_t)b * alpha_stride;
    float* deb = de + (int64_t)b * alpha_stride;
    const float* drb = dreg + (int64_t)b * dreg_stride;
    // per-row scalars (alpha, d reg) are fetched one stage ahead: a dependent global load after the warp reduction would sit on
    // the critical path of every stage
    float pa0 = 0.f, pa1 = 0.f, pd0 = 0.f, pd1 = 0.f;
    auto prefetch = [&](int i) {
      const int row = r0 + i * C::ROWS;
      const int rows = min(C::ROWS, r1 - row);
      const int ra = wid, rb = wid + AP_CWARPS;
      if (i < nst && ra < rows) {
        pa0 = alb[row + ra];
        pd0 = dreg ? drb[row + ra] : 0.f;
        if (C::RPW == 2 && rb < rows) {
          pa1 = alb[row + rb];
          pd1 = dreg ? drb[row + rb] : 0.f;
        }
      }
    };
    prefetch(0);
    for (int i = 0; i < nst; i++) {
      const int s = i % AP_STAGES;
      const uint32_t ph = (i / AP_STAGES) & 1;
      const int row = r0 + i * C::ROWS;
      const int rows = min(C::ROWS, r1 - row);
      const float al0 = pa0, al1 = pa1, dr0 = pd0, dr1 = pd1;
      prefetch(i + 1);
      mbar_wait(full_bar + s, ph);
      const T* sa = ring + (size_t)s * C::STAGE_ELEMS;
      const T* se = sa + C::HALF_A;
      const int ra = wid, rb = wid + AP_CWARPS;
      const bool one = ra < rows;
      const bool two = (C::RPW == 2) && (rb < rows);
      if (one) {
        float d0 = 0.f, d1 = 0.f;
#pragma unroll
        for (int j = 0; j < NVC; j++) {
          float u[8];
          ld8(se + (size_t)ra * CHC + (j * 32 + lane) * 8, u);
#pragma unroll
          for (int q = 0; q < 8; q++) d0 = fmaf(dc[j * 8 + q], u[q], d0);
          if (two) {
            ld8(se + (size_t)rb * CHC + (j * 32 + lane) * 8, u);
#pragma unroll
            for (int q = 0; q < 8; q++) d1 = fmaf(dc[j * 8 + q], u[q], d1);
          }
        }
        d0 = warp_sum(d0);
        d1 = warp_sum(d1);
        const float de0 = al0 * (d0 + dr0 - sall);
        const float de1 = two ? al1 * (d1 + dr1 - sall) : 0.f;
        if (lane == 0) {
          deb[row + ra] = de0;
          if (two) deb[row + rb] = de1;
        }
#pragma unroll
        for (int j = 0; j < NVA; j++) {
          float v[8], g[8], w8[8];
          const float* wj = w8;
          if constexpr (DA1 && NVA > 2) ld8(s_wf + (j * 32 + lane) * 8, w8);
          else wj = wv + j * 8;
          ld8(sa + (size_t)ra * CHA + (j * 32 + lane) * 8, v);
#pragma unroll
          for (int q = 0; q < 8; q++) {
            const float pre = v[q] + a2[j * 8 + q];
            const float post = att_act<ACT, sizeof(T) == 2>(pre);
            macc[j * 8 + q] = fmaf(de0, att_dact<ACT>(pre, post), macc[j * 8 + q]);
            wacc[j * 8 + q] = fmaf(de0, post, wacc[j * 8 + q]);
            if constexpr (DA1) g[q] = wj[q] * (de0 * att_dact<ACT>(pre, post));
          }
          if constexpr (DA1) st8(datt1 + ((int64_t)b * R + row + ra) * CHA + (j * 32 + lane) * 8, g);
          if (two) {
            ld8(sa + (size_t)rb * CHA + (j * 32 + lane) * 8, v);
#pragma unroll
            for (int q = 0; q < 8; q++) {
              const float pre = v[q] + a2[j * 8 + q];
              const float post = att_act<ACT, sizeof(T) == 2>(pre);
              macc[j * 8 + q] = fmaf(de1, att_dact<ACT>(pre, post), macc[j * 8 + q]);
              wacc[j * 8 + q] = fmaf(de1, post, wacc[j * 8 + q]);
              if constexpr (DA1) g[q] = wj[q] * (de1 * att_dact<ACT>(pre, post));
            }
            if constexpr (DA1) st8(datt1 + ((int64_t)b * R + row + rb) * CHA + (j * 32 + lane) * 8, g);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar + s);
    }
  }
  __syncthreads();
  float* s_acc = reinterpret_cast<float*>(ap_smem);            // [8][CHA] mask sums | [2][CHA] CTA totals | [8][CHA] w_full sums
  float* s_part = s_acc + AP_CWARPS * CHA;
  float* s_wacc = s_part + 2 * CHA;
  if (wid < AP_CWARPS) {
#pragma unroll
    for (int j = 0; j < NVA; j++)
#pragma unroll
      for (int i = 0; i < 8; i++) {
        s_acc[wid * CHA + (j * 32 + lane) * 8 + i] = macc[j * 8 + i];
        s_wacc[wid * CHA + (j * 32 + lane) * 8 + i] = wacc[j * 8 + i];
      }
  }
  __syncthreads();
  if constexpr (CL) {
    cg::cluster_group cluster = cg::this_cluster();
    for (int c = threadIdx.x; c < CHA; c += AP_THREADS) {
      float t = 0.f, u = 0.f;
#pragma unroll
      for (int w = 0; w < AP_CWARPS; w++) { t += s_acc[w * CHA + c]; u += s_wacc[w * CHA + c]; }
      s_part[c] = t;
      s_part[CHA + c] = u;
    }
    cluster.sync();
    const int cps = (CHA + nsplit - 1) / nsplit;
    for (int c = sp * cps + threadIdx.x; c < min(CHA, (sp + 1) * cps); c += AP_THREADS) {
      float t = 0.f, u = 0.f;
      for (int q = 0; q < nsplit; q++) {                       // fixed order -> deterministic
        const float* rp = cluster.map_shared_rank(s_part, q);
        t += rp[c];
        u += rp[CHA + c];
      }
      datt2[(int64_t)b * dcat_stride + c] = t * wf[c];
      if (datt2_bf) datt2_bf[(int64_t)b * dcat_stride + c] = __float2bfloat16_rn(t * wf[c]);
      if (dwf_part) dwf_part[(int64_t)b * CHA + c] += u;       // one writer per (b, c): plain accumulate over the time loop
    }
    cluster.sync();
    return;
  }
  if (dwf_part) {
    for (int c = threadIdx.x; c < CHA; c += AP_THREADS) {
      float u = 0.f;
#pragma unroll
      for (int w = 0; w < AP_CWARPS; w++) u += s_wacc[w * CHA + c];
      atomicAdd(dwf_part + (int64_t)b * CHA + c, u);
    }
  }
  float* part = partials + ((int64_t)b * nsplit + sp) * (CHA + 2);
  for (int c = threadIdx.x; c < CHA; c += AP_THREADS) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < AP_CWARPS; w++) t += s_acc[w * CHA + c];
    part[2 + c] = t;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int ticket = atomicAdd(counters + b, 1);
    s_last = (ticket == nsplit - 1);
    if (s_last) counters[b] = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* pb = partials + (int64_t)b * nsplit * (CHA + 2);
  for (int c = threadIdx.x; c < CHA; c += AP_THREADS) {
    float t = 0.f;
    for (int sidx = 0; sidx < nsplit; sidx++) t += __ldcg(pb + (int64_t)sidx * (CHA + 2) + 2 + c);
    datt2[(int64_t)b * dcat_stride + c] = t * wf[c];
    if (datt2_bf) datt2_bf[(int64_t)b * dcat_stride + c] = __float2bfloat16_rn(t * wf[c]);
  }
}

// ------------------------------------------------------------------------------------------------------------------------------
// Attention backward, mask-bit version (ReLU score): the forward kernel left 1 bit per att1 element (att1 + att2 > 0), so the
// backward streams enc rows (CHC elements) + CHA/8 mask bytes per region instead of enc + att1 rows: 60.5 MB instead of
// 114 MB per step at cfg #2.  Same math, same masks (the bits ARE the forward's comparisons), same combine order.
// d w_full: only its att2 term (sum_r on * de times att2) is accumulated here (dwf_part); the term that needs att1 itself is added by
// the post-loop sweep (datt1_kernel<.., WACC = 2>).
// ------------------------------------------------------------------------------------------------------------------------------
#define APM_STAGES 5
template <typename T, int NVA, int NVC>
struct ApmCfg {
  static constexpr int CHA = NVA * 256, CHC = NVC * 256;
  static constexpr int RPW = (sizeof(T) == 2 && NVC <= 2) ? LO_ATT_RPW : 1;
  static constexpr int ROWS = AP_CWARPS * RPW;
  static constexpr int ENC_BYTES = ROWS * CHC * (int)sizeof(T);
  static constexpr int MSK_BYTES = ROWS * (CHA / 8);
  static constexpr int STAGE_BYTES = ENC_BYTES + MSK_BYTES;
  static constexpr int SMEM = APM_STAGES * STAGE_BYTES + 128;
  static_assert(APM_STAGES * STAGE_BYTES >= (AP_CWARPS + 2) * CHA * 4, "combine scratch must fit in the ring");
};

template <typename T, int NVA, int NVC, bool CL>
__global__ void __launch_bounds__(AP_THREADS, LO_ATT_MINB) attention_bwd_mask_kernel(
    const uint8_t* __restrict__ mask, const T* __restrict__ enc, const float* __restrict__ gate, int64_t o1_stride,
    const float* __restrict__ wf, const float* __restrict__ alpha, int64_t alpha_stride, const float* __restrict__ ctx,
    const float* __restrict__ dgctx, int64_t dg_stride, const float* __restrict__ dreg, int64_t dreg_stride,
    const float* __restrict__ sreg, int64_t sreg_stride, float* __restrict__ de, float* __restrict__ datt2, float* __restrict__ dgp,
    int64_t dcat_stride, bf16* __restrict__ datt2_bf, bf16* __restrict__ dgp_bf, float* __restrict__ dctx_out, int R, int nsplit,
    int* __restrict__ counters, float* __restrict__ partials, const float* __restrict__ att2, float* __restrict__ dwf_part) {
  using C = ApmCfg<T, NVA, NVC>;
  constexpr int CHA = C::CHA, CHC = C::CHC, MB = CHA / 8;
  extern __shared__ __align__(128) uint8_t ap_smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ap_smem + APM_STAGES * C::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + APM_STAGES;
  __shared__ int s_last;
  const int b = blockIdx.y, sp = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int rps = att_rows_per_split(R, nsplit);          // even (and ROWS is even): stages start on an (even, odd) row pair
  const int r0 = sp * rps, r1 = min(R, r0 + rps);
  const int nst = r1 > r0 ? (r1 - r0 + C::ROWS - 1) / C::ROWS : 0;
  const T* eb = enc + (int64_t)b * R * CHC;
  const uint8_t* mb = mask + (int64_t)b * ((R + 1) & ~1) * MB;      // pair layout, see attention_fwd_pipe_kernel
  if (threadIdx.x == 0) {
    for (int s = 0; s < APM_STAGES; s++) {
      mbar_init(full_bar + s, 1);
      mbar_init(empty_bar + s, AP_CWARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  float macc[NVA * 8];
#pragma unroll
  for (int i = 0; i < NVA * 8; i++) macc[i] = 0.f;

  if (wid == AP_CWARPS) {
    // producer: enc is loop-invariant (prefetchable before griddepcontrol.wait); the mask bits of this step were written by the
    // forward pass long ago as well
    if (lane == 0) {
      const uint64_t pe = l2_policy_evict_last(), pm = l2_policy_evict_first();
      for (int i = 0; i < nst; i++) {
        const int s = i % APM_STAGES;
        const uint32_t ph = (i / APM_STAGES) & 1;
        mbar_wait(empty_bar + s, ph ^ 1);
        const int row = r0 + i * C::ROWS;
        const int rows = min(C::ROWS, r1 - row);
        const uint32_t bytes_c = (uint32_t)rows * CHC * (uint32_t)sizeof(T), bytes_m = (uint32_t)((rows + 1) >> 1) * 2u * MB;
        uint8_t* st = ap_smem + (size_t)s * C::STAGE_BYTES;
        mbar_expect_tx(full_bar + s, bytes_c + bytes_m);
        bulk_g2s(st, eb + (int64_t)row * CHC, bytes_c, full_bar + s, pe);
        bulk_g2s(st + C::ENC_BYTES, mb + (int64_t)row * MB, bytes_m, full_bar + s, pm);
      }
    }
    __syncwarp();
    pdl_wait();
  } else {
    float dc[NVC * 8];
    float sdot = 0.f;
    float gv[NVC * 8], cxv[NVC * 8];
#pragma unroll
    for (int j = 0; j < NVC; j++) {
      const int c0 = (j * 32 + lane) * 8;
      if (gate) ld8(gate + (int64_t)b * o1_stride + c0, gv + j * 8);
      ld8(ctx + (int64_t)b * CHC + c0, cxv + j * 8);
    }
    const float sreg_b = sreg ? sreg[(int64_t)b * sreg_stride] : 0.f;
    pdl_wait();
    pdl_trigger();
#pragma unroll
    for (int j = 0; j < NVC; j++) {
      const int c0 = (j * 32 + lane) * 8;
      float dg[8], gp[8];
      ld8(dgctx + (int64_t)b * dg_stride + c0, dg);
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const float gi = gate ? gv[j * 8 + i] : 1.f;
        dc[j * 8 + i] = dg[i] * gi;
        sdot = fmaf(dc[j * 8 + i], cxv[j * 8 + i], sdot);
        gp[i] = dg[i] * cxv[j * 8 + i] * gi * (1.f - gi);
      }
      if (sp == 0 && wid == 0) {
        if (dgp) st8(dgp + (int64_t)b * dcat_stride + c0, gp);
        if (dgp_bf) st8(dgp_bf + (int64_t)b * dcat_stride + c0, gp);
        if (dctx_out) st8(dctx_out + (int64_t)b * CHC + c0, dc + j * 8);
      }
    }
    const float sall = warp_sum(sdot) + sreg_b;
    const float* alb = alpha + (int64_t)b * alpha_stride;
    float* deb = de + (int64_t)b * alpha_stride;
    const float* drb = dreg + (int64_t)b * dreg_stride;
    float pa0 = 0.f, pa1 = 0.f, pd0 = 0.f, pd1 = 0.f;
    auto prefetch = [&](int i) {
      const int row = r0 + i * C::ROWS;
      const int rows = min(C::ROWS, r1 - row);
      const int ra = wid, rb = wid + AP_CWARPS;
      if (i < nst && ra < rows) {
        pa0 = alb[row + ra];
        pd0 = dreg ? drb[row + ra] : 0.f;
        if (C::RPW == 2 && rb < rows) {
          pa1 = alb[row + rb];
          pd1 = dreg ? drb[row + rb] : 0.f;
        }
      }
    };
    prefetch(0);
    for (int i = 0; i < nst; i++) {
      const int s = i % APM_STAGES;
      const uint32_t ph = (i / APM_STAGES) & 1;
      const int row = r0 + i * C::ROWS;
      const int rows = min(C::ROWS, r1 - row);
      const float al0 = pa0, al1 = pa1, dr0 = pd0, dr1 = pd1;
      prefetch(i + 1);
      mbar_wait(full_bar + s, ph);
      const uint32_t se = smem_u32(ap_smem + (size_t)s * C::STAGE_BYTES);
      constexpr uint32_t ES = (uint32_t)sizeof(T);
      const uint8_t* sm = ap_smem + (size_t)s * C::STAGE_BYTES + C::ENC_BYTES;
      const int ra = wid, rb = wid + AP_CWARPS;
      const bool one = ra < rows;
      const bool two = (C::RPW == 2) && (rb < rows);
      if (one) {
        float d0 = 0.f, d1 = 0.f;
#pragma unroll
        for (int j = 0; j < NVC; j++) {
          float u[8];
          lds8(se + ((uint32_t)ra * CHC + (j * 32 + lane) * 8) * ES, u, (const T*)nullptr);
#pragma unroll
          for (int q = 0; q < 8; q++) d0 = fmaf(dc[j * 8 + q], u[q], d0);
          if (two) {
            lds8(se + ((uint32_t)rb * CHC + (j * 32 + lane) * 8) * ES, u, (const T*)nullptr);
#pragma unroll
            for (int q = 0; q < 8; q++) d1 = fmaf(dc[j * 8 + q], u[q], d1);
          }
        }
        d0 = warp_sum(d0);
        d1 = warp_sum(d1);
        const float de0 = al0 * (d0 + dr0 - sall);
        const float de1 = two ? al1 * (d1 + dr1 - sall) : 0.f;
        if (lane == 0) {
          deb[row + ra] = de0;
          if (two) deb[row + rb] = de1;
        }
#pragma unroll
        for (int j = 0; j < NVA; j++) {
          const uint32_t m0 = sm[(ra >> 1) * 2 * MB + (j * 32 + lane) * 2 + (ra & 1)];
          const uint32_t m1 = two ? sm[(rb >> 1) * 2 * MB + (j * 32 + lane) * 2 + (rb & 1)] : 0u;
#pragma unroll
          for (int q = 0; q < 8; q++) {
            if (m0 & (0x80u >> q)) macc[j * 8 + q] += de0;
            if (m1 & (0x80u >> q)) macc[j * 8 + q] += de1;
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar + s);
    }
  }
  __syncthreads();
  float* s_acc = reinterpret_cast<float*>(ap_smem);            // [8][CHA] mask sums | [CHA] CTA totals
  float* s_part = s_acc + AP_CWARPS * CHA;
  if (wid < AP_CWARPS) {
#pragma unroll
    for (int j = 0; j < NVA; j++)
#pragma unroll
      for (int i = 0; i < 8; i++) s_acc[wid * CHA + (j * 32 + lane) * 8 + i] = macc[j * 8 + i];
  }
  __syncthreads();
  if constexpr (CL) {
    cg::cluster_group cluster = cg::this_cluster();
    for (int c = threadIdx.x; c < CHA; c += AP_THREADS) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < AP_CWARPS; w++) t += s_acc[w * CHA + c];
      s_part[c] = t;
    }
    cluster.sync();
    const int cps = (CHA + nsplit - 1) / nsplit;
    for (int c = sp * cps + threadIdx.x; c < min(CHA, (sp + 1) * cps); c += AP_THREADS) {
      float t = 0.f;
      for (int q = 0; q < nsplit; q++) t += cluster.map_shared_rank(s_part, q)[c];      // fixed order -> deterministic
      if (dwf_part) dwf_part[(int64_t)b * CHA + c] += t * att2[(int64_t)b * o1_stride + c];    // att2 term of d w_full (one owner per (b, c))
      datt2[(int64_t)b * dcat_stride + c] = t * wf[c];
      if (datt2_bf) datt2_bf[(int64_t)b * dcat_stride + c] = __float2bfloat16_rn(t * wf[c]);
    }
    cluster.sync();
    return;
  }
  float* part = partials + ((int64_t)b * nsplit + sp) * (CHA + 2);
  for (int c = threadIdx.x; c < CHA; c += AP_THREADS) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < AP_CWARPS; w++) t += s_acc[w * CHA + c];
    part[2 + c] = t;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int ticket = atomicAdd(counters + b, 1);
    s_last = (ticket == nsplit - 1);
    if (s_last) counters[b] = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* pb = partials + (int64_t)b * nsplit * (CHA + 2);
  for (int c = threadIdx.x; c < CHA; c += AP_THREADS) {
    float t = 0.f;
    for (int sidx = 0; sidx < nsplit; sidx++) t += __ldcg(pb + (int64_t)sidx * (CHA + 2) + 2 + c);
    if (dwf_part) dwf_part[(int64_t)b * CHA + c] += t * att2[(int64_t)b * o1_stride + c];
    datt2[(int64_t)b * dcat_stride + c] = t * wf[c];
    if (datt2_bf) datt2_bf[(int64_t)b * dcat_stride + c] = __float2bfloat16_rn(t * wf[c]);
  }
}

// ------------------------------------------------------------------------------------------------------------------------------
// [r2b] Tensor-core backward for the 512-wide torch flavour (bf16): the two contractions of the step run on mma.sync instead of
// CUDA-core FMAs / predicated adds (2.5x fewer warp instructions).  The launch is not issue-bound — what it loses it loses at its
// ends — but the tensor-core version frees the issue slots, and alpha / d reg are staged in shared memory and the tail operands
// fetched up front:
//   d[r]     = sum_c enc[r][c] * dctx[c]          A = 16 enc rows straight from the ring (ldmatrix), B = dctx split into bf16 hi+lo
//                                                  (columns 0/1 of B, products exact, fp32 accumulation)
//   datt2[a] = sum_r bit[r][a] * de[r]            A = mask bits expanded to bf16 {0, 2.0} with ONE shift + ONE and per register,
//                                                  B = de split into bf16 hi+lo
// A stage is 16 region rows; all 8 consumer warps share it: warp w takes channels [64w, 64w+64) of the dot product (4 k-steps),
// the 16 partial sums per warp meet in shared memory behind one 256-thread named barrier, every warp then forms de for the 16
// rows (redundantly: 16 lanes) and runs the mask contraction for ITS 64 attention columns (4 blocks of 16).  ~110 warp
// instructions per warp and stage instead of ~260 per 2 rows.
// Ring rows are padded to 1040 B (one bulk copy per row) so that the 8 rows of an ldmatrix phase hit 8 different 16-byte bank
// groups.  Mask layout (written by the forward kernel): byte (r, a/8) lives at (r/2) * 2*(A/8) + (a/8)*2 + (r&1), i.e. the bytes
// of an even/odd row pair are adjacent: a lane's four A registers per 16 x 16 block are then shifts of ONE 32-bit word
// [even(q) | even(q+4) | odd(q) | odd(q+4)] (q = lane % 4: fragment k index = region row).  Fragment row m = g + 8h of block j
// stands for attention column 64w + 8g + 2j + h (g = lane / 4): any bijection works, this one makes a lane's 8 columns one byte.
// ------------------------------------------------------------------------------------------------------------------------------
// Ring depth and CTAs per SM.  The grid is one wave at 2 CTAs per SM (att_pipe_splits: 4 splits at B = 64).  On the H100 a
// one-wave grid of 4-CTA clusters with exactly 2 slots per SM did not become resident at once: about an eighth of the CTAs entered
// only when others exited and the launch ended in a second wave of full-length CTAs.  With clusters, a 3-stage ring that lets 3
// CTAs share an SM was the cure (backward time loop at B = 64, H100 SXM, 400 W, us per step: 5 stages / 2 per SM 53.2, 4 / 3 48.0,
// 3 / 3 47.6).  The default launch has no cluster (att_grid_cluster): 256 independent CTAs fill 264 slots, and the deeper ring at
// 2 per SM wins (same card, cluster-free: 3 / 3 45.4, 4 / 2 42.8, 5 / 2 41.7).
#ifndef LO_ABM_STAGES
#define LO_ABM_STAGES 5
#endif
#ifndef LO_ABM_MINB
#define LO_ABM_MINB 2
#endif
constexpr int ABM_STAGES = LO_ABM_STAGES;
constexpr int ABM_ROWS = 16;
constexpr int ABM_CH = 512;
constexpr int ABM_PITCH = ABM_CH * 2 + 16;                    // bytes per ring row
constexpr int ABM_ENC_BYTES = ABM_ROWS * ABM_PITCH;
constexpr int ABM_MSK_BYTES = ABM_ROWS * (ABM_CH / 8);
constexpr int ABM_STAGE_BYTES = ABM_ENC_BYTES + ABM_MSK_BYTES;
constexpr int ABM_SMEM = ABM_STAGES * ABM_STAGE_BYTES + 128 + 2 * AP_CWARPS * ABM_ROWS * 4;
static_assert(ABM_STAGE_BYTES % 128 == 0, "stage alignment");

__device__ __forceinline__ void att_ldsm_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(saddr));
}
__device__ __forceinline__ void att_mma_16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// (x, y) -> packed bf16 pair of the high parts (sel 0) or of the residuals x - hi(x) (sel 1); low half = x
__device__ __forceinline__ uint32_t pack_split(float x, float y, int sel) {
  const bf16 hx = __float2bfloat16_rn(x), hy = __float2bfloat16_rn(y);
  __nv_bfloat162 r;
  if (sel == 0) {
    r.x = hx; r.y = hy;
  } else {
    r.x = __float2bfloat16_rn(x - __bfloat162float(hx));
    r.y = __float2bfloat16_rn(y - __bfloat162float(hy));
  }
  return *reinterpret_cast<uint32_t*>(&r);
}

template <bool CL>
__global__ void __launch_bounds__(AP_THREADS, LO_ABM_MINB) attention_bwd_mma_kernel(
    const uint8_t* __restrict__ mask, const bf16* __restrict__ enc, const float* __restrict__ gate, int64_t o1_stride,
    const float* __restrict__ wf, const float* __restrict__ alpha, int64_t alpha_stride, const float* __restrict__ ctx,
    const float* __restrict__ dgctx, int64_t dg_stride, const float* __restrict__ dreg, int64_t dreg_stride,
    const float* __restrict__ sreg, int64_t sreg_stride, float* __restrict__ de, float* __restrict__ datt2, float* __restrict__ dgp,
    int64_t dcat_stride, bf16* __restrict__ datt2_bf, bf16* __restrict__ dgp_bf, float* __restrict__ dctx_out, int R, int nsplit,
    int* __restrict__ counters, float* __restrict__ partials, int keep_q, const float* __restrict__ att2,
    float* __restrict__ dwf_part) {
  constexpr int CH = ABM_CH, MB = CH / 8;
  extern __shared__ __align__(128) uint8_t ap_smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ap_smem + ABM_STAGES * ABM_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + ABM_STAGES;
  float* s_pd = reinterpret_cast<float*>(ap_smem + ABM_STAGES * ABM_STAGE_BYTES + 128);      // [2][8 warps][16 rows] partial dots
  __shared__ int s_last;
  const int b = blockIdx.y, sp = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int rps = att_rows_per_split(R, nsplit);                // even: a stage starts on an even/odd row pair
  const int r0 = sp * rps, r1 = min(R, r0 + rps);
  const int nst = r1 > r0 ? (r1 - r0 + ABM_ROWS - 1) / ABM_ROWS : 0;
  const int Rp = (R + 1) & ~1;
  ATT_TS(0, threadIdx.x == 0);
  const bf16* eb = enc + (int64_t)b * R * CH;
  const uint8_t* mb = mask + (int64_t)b * Rp * MB;
  if (threadIdx.x == 0) {
    for (int s = 0; s < ABM_STAGES; s++) {
      mbar_init(full_bar + s, 1);
      mbar_init(empty_bar + s, AP_CWARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int g = lane >> 2, q = lane & 3;
  // cluster mode: the full_att weight and the att2 value of the column this thread finalises after the combine are forward-pass
  // data -> fetched up front, off the tail
  const int cps_pf = (CH + nsplit - 1) / nsplit;
  const int c_pf = sp * cps_pf + (int)threadIdx.x;
  float wf_pf = 0.f, a2_pf = 0.f;
  if (CL && (int)threadIdx.x < cps_pf && c_pf < CH) {
    wf_pf = wf[c_pf];
    if (dwf_part) a2_pf = att2[(int64_t)b * o1_stride + c_pf];
  }
  float macc[4][4];
#pragma unroll
  for (int j = 0; j < 4; j++)
#pragma unroll
    for (int i = 0; i < 4; i++) macc[j][i] = 0.f;

  if (wid == AP_CWARPS) {
    // producer warp: enc and the mask bits of this step were written long before the preceding launch -> no griddepcontrol.wait
    // the whole budget goes to enc rows; the mask bits of a step are read once per time loop
    const uint64_t pk = l2_policy_evict_normal(), pm = l2_policy_evict_first();
    for (int i = 0; i < nst; i++) {
      const int s = i % ABM_STAGES;
      const uint32_t ph = (i / ABM_STAGES) & 1;
      const int row = r0 + i * ABM_ROWS;
      const int rows = min(ABM_ROWS, r1 - row);
      const uint32_t bytes_m = (uint32_t)((rows + 1) >> 1) * 2u * MB;
      uint8_t* st = ap_smem + (size_t)s * ABM_STAGE_BYTES;
      if (lane == 0) {
        mbar_wait(empty_bar + s, ph ^ 1);
        mbar_expect_tx(full_bar + s, (uint32_t)rows * CH * 2u + bytes_m);
        ATT_TS(6, i == 0);
        ATT_TS(7, i == nst - 1);
      }
      __syncwarp();
      const uint64_t pe = att_keep_stage(i, ABM_STAGES, keep_q) ? pk : pm;
      if (lane < rows) bulk_g2s(st + lane * ABM_PITCH, eb + (int64_t)(row + lane) * CH, CH * 2u, full_bar + s, pe);
      else if (lane == ABM_ROWS) bulk_g2s(st + ABM_ENC_BYTES, mb + (int64_t)(row >> 1) * 2 * MB, bytes_m, full_bar + s, pm);
    }
    __syncwarp();
    pdl_wait();
  } else {
    float sdot = 0.f;
    float gv[16], cxv[16];
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const int c0 = (j * 32 + lane) * 8;
      if (gate) ld8(gate + (int64_t)b * o1_stride + c0, gv + j * 8);
      ld8(ctx + (int64_t)b * CH + c0, cxv + j * 8);
    }
    // this lane's slice of the B operand of the dot product: k = 64*wid + 16*s + 2q + {0,1,8,9}; columns 0 / 1 = hi / lo parts
    float gq[4][4];
#pragma unroll
    for (int s = 0; s < 4; s++) {
      const int k0 = 64 * wid + 16 * s + 2 * q;
      if (gate && g < 2) {
        const float2 u = *reinterpret_cast<const float2*>(gate + (int64_t)b * o1_stride + k0);
        const float2 v = *reinterpret_cast<const float2*>(gate + (int64_t)b * o1_stride + k0 + 8);
        gq[s][0] = u.x; gq[s][1] = u.y; gq[s][2] = v.x; gq[s][3] = v.y;
      } else {
        gq[s][0] = gq[s][1] = gq[s][2] = gq[s][3] = 1.f;
      }
    }
    const float sreg_b = sreg ? sreg[(int64_t)b * sreg_stride] : 0.f;
    // alpha and the regulariser gradient of this CTA's rows are forward-pass results: ALL of them are staged in shared memory before
    // the wait.  (Fetching them stage by stage with a one-stage lookahead makes every 16-row stage cost one L2 round trip, which then
    // bounds the main loop whatever the arithmetic is.)
    const float* alb = alpha + (int64_t)b * alpha_stride;
    float* deb = de + (int64_t)b * alpha_stride;
    const float* drb = dreg + (int64_t)b * dreg_stride;
    const int rr = lane & 15;
    float* s_al = s_pd + 2 * AP_CWARPS * ABM_ROWS;      // [rps] alpha | [rps] d reg
    float* s_dr = s_al + rps;
    for (int r = threadIdx.x; r < r1 - r0; r += AP_CWARPS * 32) {
      s_al[r] = alb[r0 + r];
      s_dr[r] = dreg ? drb[r0 + r] : 0.f;
    }
    pdl_wait();
    ATT_TS(1, threadIdx.x == 0);
    pdl_trigger();
    uint32_t bd[4][2];
#pragma unroll
    for (int s = 0; s < 4; s++) {
      bd[s][0] = bd[s][1] = 0u;
      if (g < 2) {
        const int k0 = 64 * wid + 16 * s + 2 * q;
        const float2 u = *reinterpret_cast<const float2*>(dgctx + (int64_t)b * dg_stride + k0);
        const float2 v = *reinterpret_cast<const float2*>(dgctx + (int64_t)b * dg_stride + k0 + 8);
        bd[s][0] = pack_split(u.x * gq[s][0], u.y * gq[s][1], g);
        bd[s][1] = pack_split(v.x * gq[s][2], v.y * gq[s][3], g);
      }
    }
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const int c0 = (j * 32 + lane) * 8;
      float dg[8], gp[8], dc[8];
      ld8(dgctx + (int64_t)b * dg_stride + c0, dg);
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const float gi = gate ? gv[j * 8 + i] : 1.f;
        dc[i] = dg[i] * gi;
        sdot = fmaf(dc[i], cxv[j * 8 + i], sdot);
        gp[i] = dg[i] * cxv[j * 8 + i] * gi * (1.f - gi);
      }
      if (sp == 0 && wid == 0) {
        if (dgp) st8(dgp + (int64_t)b * dcat_stride + c0, gp);
        if (dgp_bf) st8(dgp_bf + (int64_t)b * dcat_stride + c0, gp);
        if (dctx_out) st8(dctx_out + (int64_t)b * CH + c0, dc);
      }
    }
    const float sall = warp_sum(sdot) + sreg_b;
    ATT_TS(2, threadIdx.x == 0);
    const uint32_t ring = smem_u32(ap_smem);
    const uint32_t a_off = (uint32_t)((lane & 7) + ((lane >> 3) & 1) * 8) * ABM_PITCH + (uint32_t)(64 * wid + (lane >> 4) * 8) * 2u;
    const uint32_t m_off = ABM_ENC_BYTES + (uint32_t)q * 2u * MB + (uint32_t)(8 * wid + g) * 2u;
    asm volatile("bar.sync 1, 256;" ::: "memory");     // s_al / s_dr complete
    for (int i = 0; i < nst; i++) {
      const int s = i % ABM_STAGES;
      const uint32_t ph = (i / ABM_STAGES) & 1;
      const int row = r0 + i * ABM_ROWS;
      const int rows = min(ABM_ROWS, r1 - row);
      const float al = rr < rows ? s_al[i * ABM_ROWS + rr] : 0.f, dr = rr < rows ? s_dr[i * ABM_ROWS + rr] : 0.f;
      mbar_wait(full_bar + s, ph);
      ATT_TS(3, threadIdx.x == 0 && i == 0);
      const uint32_t sb = ring + (uint32_t)s * ABM_STAGE_BYTES;
      // ---- partial dot products of the 16 rows over this warp's 64 channels
      float d4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < 4; k++) {
        uint32_t a0, a1, a2, a3;
        att_ldsm_x4(a0, a1, a2, a3, sb + a_off + k * 32);
        att_mma_16816(d4, a0, a1, a2, a3, bd[k][0], bd[k][1]);
      }
      // this lane's mask word (read now: the ring slot is released right after the barrier-independent part)
      const uint32_t u_lo = *reinterpret_cast<const uint16_t*>(ap_smem + (size_t)s * ABM_STAGE_BYTES + m_off);
      const uint32_t u_hi = *reinterpret_cast<const uint16_t*>(ap_smem + (size_t)s * ABM_STAGE_BYTES + m_off + 4 * 2 * MB);
      const uint32_t mw = __byte_perm(u_lo, u_hi, 0x5140);      // [even(q) | even(q+4) | odd(q) | odd(q+4)]
      float* pdw = s_pd + (i & 1) * (AP_CWARPS * ABM_ROWS);
      if (q == 0) {
        pdw[wid * ABM_ROWS + g] = d4[0] + d4[1];
        pdw[wid * ABM_ROWS + g + 8] = d4[2] + d4[3];
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar + s);                 // every lane of this warp has read what it needs from the slot
      asm volatile("bar.sync 1, 256;" ::: "memory");
      float dsum = 0.f;
#pragma unroll
      for (int w = 0; w < AP_CWARPS; w++) dsum += pdw[w * ABM_ROWS + rr];
      const float dev = rr < rows ? al * (dsum + dr - sall) : 0.f;
      if (wid == (i & 7) && lane < rows) deb[row + lane] = dev;
      // ---- mask contraction: B = de of rows (2q, 2q+1, 2q+8, 2q+9), hi parts in column 0 (g == 0), residuals in column 1
      const float v0 = __shfl_sync(0xffffffffu, dev, 2 * q), v1 = __shfl_sync(0xffffffffu, dev, 2 * q + 1);
      const float v2 = __shfl_sync(0xffffffffu, dev, 2 * q + 8), v3 = __shfl_sync(0xffffffffu, dev, 2 * q + 9);
      uint32_t bm0 = 0u, bm1 = 0u;
      if (g < 2) {
        bm0 = pack_split(v0, v1, g);
        bm1 = pack_split(v2, v3, g);
      }
#pragma unroll
      for (int j = 0; j < 4; j++) {
        uint32_t af[4];
#pragma unroll
        for (int ii = 0; ii < 4; ii++) {
          // element e=0 (low half): bit 8*rs + 7 - (2j + h); e=1: 16 above.  -> bit 14 / 30 (bf16 2.0)
          const int h = ii & 1, rs = ii >> 1;
          const int sh = 14 - (8 * rs + 7 - (2 * j + h));
          af[ii] = (sh >= 0 ? (mw << sh) : (mw >> (-sh))) & 0x40004000u;
        }
        att_mma_16816(macc[j], af[0], af[1], af[2], af[3], bm0, bm1);
      }
    }
  }
  ATT_TS(4, threadIdx.x == 0);
  // cluster-free: full_att weight, att2 and the running d w_full sum of the columns this thread finalises should its CTA combine
  // last (column c = tid + k * AP_THREADS, below): fetched now, behind the CTA combine and the ticket.  Only the last CTA of this
  // batch row writes its d w_full row, after its ticket.
  constexpr int NCB = (CH + AP_THREADS - 1) / AP_THREADS;
  float wf_t[NCB], a2_t[NCB], dwf_t[NCB];
  if constexpr (!CL) {
#pragma unroll
    for (int k = 0; k < NCB; k++) {
      const int c = threadIdx.x + k * AP_THREADS;
      wf_t[k] = c < CH ? wf[c] : 0.f;
      a2_t[k] = (dwf_part && c < CH) ? att2[(int64_t)b * o1_stride + c] : 0.f;
      dwf_t[k] = (dwf_part && c < CH) ? dwf_part[(int64_t)b * CH + c] : 0.f;
    }
  }
  __syncthreads();
  ATT_TS(8, threadIdx.x == 0);
  float* s_part = reinterpret_cast<float*>(ap_smem);             // [CH] mask sums of this CTA (every column has ONE owner lane)
  if (wid < AP_CWARPS && q == 0) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      s_part[64 * wid + 8 * g + 2 * j] = 0.5f * (macc[j][0] + macc[j][1]);
      s_part[64 * wid + 8 * g + 2 * j + 1] = 0.5f * (macc[j][2] + macc[j][3]);
    }
  }
  __syncthreads();
  if constexpr (CL) {
    cg::cluster_group cluster = cg::this_cluster();
    // the running d w_full sum of this thread's column (last written by an earlier step): its load overlaps the cluster barrier
    const float dwf_pf = dwf_part && (int)threadIdx.x < cps_pf && c_pf < CH ? dwf_part[(int64_t)b * CH + c_pf] : 0.f;
    cluster.sync();
    const int cps = (CH + nsplit - 1) / nsplit;
    // gather the peers' sums first (into the ring behind s_part, which no peer reads), arrive, then the global read-modify-writes
    // overlap the barrier
    float* s_sum = s_part + CH;
    for (int c = sp * cps + threadIdx.x; c < min(CH, (sp + 1) * cps); c += AP_THREADS) {
      float t = 0.f;
      for (int qq = 0; qq < nsplit; qq++) t += cluster.map_shared_rank(s_part, qq)[c];      // fixed order -> deterministic
      s_sum[c - sp * cps] = t;
    }
    cl_arrive_release();
    for (int c = sp * cps + threadIdx.x; c < min(CH, (sp + 1) * cps); c += AP_THREADS) {
      const float t = s_sum[c - sp * cps];
      const bool pf = c == c_pf;
      const float wfc = pf ? wf_pf : wf[c];
      if (dwf_part)      // att2 term of d w_full (one owner per (b, c))
        dwf_part[(int64_t)b * CH + c] = (pf ? dwf_pf : dwf_part[(int64_t)b * CH + c]) + t * (pf ? a2_pf : att2[(int64_t)b * o1_stride + c]);
      datt2[(int64_t)b * dcat_stride + c] = t * wfc;
      if (datt2_bf) datt2_bf[(int64_t)b * dcat_stride + c] = __float2bfloat16_rn(t * wfc);
    }
    cl_wait_acquire();                                           // peers may still be reading this CTA's s_part
    ATT_TS(5, threadIdx.x == 0);
    return;
  }
  float* part = partials + ((int64_t)b * nsplit + sp) * (CH + 2);
  for (int c = threadIdx.x; c < CH; c += AP_THREADS) part[2 + c] = s_part[c];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int ticket = atomicAdd(counters + b, 1);
    s_last = (ticket == nsplit - 1);
    if (s_last) counters[b] = 0;
  }
  __syncthreads();
  if (!s_last) {
    ATT_TS(5, threadIdx.x == 0);
    return;
  }
  __threadfence();
  ATT_TS(9, threadIdx.x == 0);
  // ordered combine, split order 0..nsplit-1 as in the cluster combine; the partial sums of a column are loaded together
  const float* pb = partials + (int64_t)b * nsplit * (CH + 2);
  constexpr int PS = 8;
#pragma unroll
  for (int k = 0; k < NCB; k++) {
    const int c = threadIdx.x + k * AP_THREADS;
    if (c < CH) {
      float pv[PS];
#pragma unroll
      for (int s = 0; s < PS; s++) pv[s] = s < nsplit ? __ldcg(pb + (int64_t)s * (CH + 2) + 2 + c) : 0.f;
      float t = 0.f;
#pragma unroll
      for (int s = 0; s < PS; s++)
        if (s < nsplit) t += pv[s];
      for (int s = PS; s < nsplit; s++) t += __ldcg(pb + (int64_t)s * (CH + 2) + 2 + c);
      if (dwf_part) dwf_part[(int64_t)b * CH + c] = dwf_t[k] + t * a2_t[k];
      datt2[(int64_t)b * dcat_stride + c] = t * wf_t[k];
      if (datt2_bf) datt2_bf[(int64_t)b * dcat_stride + c] = __float2bfloat16_rn(t * wf_t[k]);
    }
  }
  ATT_TS(5, threadIdx.x == 0);
}

int att_pipe_splits(int B, int hint = 0) {
  if (g_opt_att_nsplit > 0) return g_opt_att_nsplit > AP_MAXSPLIT ? AP_MAXSPLIT : g_opt_att_nsplit;      // explicit option wins
  if (hint > 0) return hint > 8 ? 8 : hint;
  // two CTAs per SM are resident (smem): aim for one full wave — per-CTA start-up/combine costs dominate short CTAs
  int s = (LO_NUM_SMS * LO_ATT_MINB) / B;
  if (s < 1) s = 1;
  if (s > AP_MAXSPLIT) s = AP_MAXSPLIT;
  if (g_opt_att_cluster && s > 8) s = 8;       // portable cluster size limit
  return s;
}

// Keep share (1/1024 units, att_keep_stage) of a launch whose CTAs stream `bytes` distinct bytes of att1 / enc rows: the
// att_l2_keep_mb budget, clamped to the device's L2 size, over those bytes.  A CTA keeps at most that share of its stages after the
// first `depth`, and all but its last stage are full, so the kept bytes of the launch never exceed the budget.
static int att_keep_q(int64_t bytes) {
  static const int64_t l2_bytes = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, dev) != cudaSuccess) {
      cudaGetLastError();
      return (int64_t)0;         // unknown: keep nothing
    }
    return (int64_t)v;
  }();
  int64_t budget = (int64_t)g_opt_att_l2_keep_mb << 20;
  if (budget > l2_bytes) budget = l2_bytes;
  if (budget <= 0 || bytes <= 0) return 0;
  const int64_t q = budget * 1024 / bytes;
  return q > 1024 ? 1024 : (int)q;
}

// optional L2 access-policy window attached to every attention launch (lo_set_l2_window): as a LAUNCH attribute it is also
// recorded in CUDA-graph kernel nodes, which a stream attribute is not
static cudaAccessPolicyWindow g_att_window{};

static inline bool att_pdl_ok(int abi) { return !abi || g_opt_att_abi_pdl; }

// launch with (optional) cluster dimension {ns,1,1} and the PDL attribute.
// pdl = false (stand-alone C entry points): these kernels read operands BEFORE griddepcontrol.wait — loop-invariant inputs in the
// forward (att1, enc, full_att weight), forward-pass results in the backward (alpha, ctx, gate, att2, d reg).  Inside the decoder's
// time loops those are at least two launches old; a caller of the C ABI may have produced them with the launch enqueued just before,
// which would be allowed to overlap.  Without the attribute the launch is fully stream-ordered (the wait is a no-op).
template <typename... KArgs, typename... Args>
static cudaError_t launch_att(void (*kernel)(KArgs...), dim3 grid, size_t smem, int cluster_x, cudaStream_t st, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(AP_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[3];
  int n = 0;
  if (g_att_window.num_bytes) {
    attr[n].id = cudaLaunchAttributeAccessPolicyWindow;
    attr[n].val.accessPolicyWindow = g_att_window;
    n++;
  }
  if (g_opt_pdl && pdl) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    n++;
  }
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    n++;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

static inline bool use_cluster(int ns, int R) {
  // cluster mode keeps the raw scores of a CTA's rows in shared memory: ceil(R/ns) floats next to the ring
  return g_opt_att_cluster && ns >= 2 && ns <= 8 && ((R + ns - 1) / ns) * 4 <= 16 * 1024;
}

// Resident CTAs of `kernel` at `smem` bytes of dynamic shared memory on the whole device.  Queried once per (device, kernel,
// shared memory) and cached: the launch paths call this on every step, also while a CUDA graph is being captured.
static int att_resident_ctas(const void* kernel, size_t smem) {
  struct Entry { int dev; const void* k; size_t smem; int ctas; };
  static std::mutex mu;
  static std::vector<Entry> cache;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  std::lock_guard<std::mutex> lock(mu);
  for (const Entry& e : cache)
    if (e.dev == dev && e.k == kernel && e.smem == smem) return e.ctas;
  int per_sm = 0, sms = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, AP_THREADS, smem) != cudaSuccess ||
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
    cudaGetLastError();
    return 0;                    // unknown: the caller keeps the cluster launch
  }
  cache.push_back({dev, kernel, smem, per_sm * sms});
  return per_sm * sms;
}

// Grid choice of the forward pipe kernel and the tensor-core backward (att_cluster): 2 always launches the splits of a batch row as
// a thread-block cluster, 0 never; 1 (default) launches without a cluster whenever the cluster-free grid of ns * B CTAs is one
// resident wave.  Both combines add the nsplit partials in split order with the same operations, so the choice changes timing only.
// Why: cluster placement could not fill the last slots of a 2-CTA-per-SM grid (4 x 64 CTAs in 2 x 132 slots on the H100), and
// about an eighth of the CTAs ran as a second wave; 256 independent CTAs are all resident at launch.
static bool att_grid_cluster(const void* free_kernel, size_t free_smem, int ns, int B, int R) {
  if (!use_cluster(ns, R)) return false;
  if (g_opt_att_cluster != 1) return true;
  return att_resident_ctas(free_kernel, free_smem) < ns * B;
}

template <typename T, int NVA, int NVC, int ACT, bool MK>
static int fwd_launch_m(const AttFwdArgs& x, cudaStream_t st) {
  using C = ApCfg<T, NVA, NVC>;
  constexpr int SM_MAX = C::SMEM + 16 * 1024;
  static bool attr = false;
  if (!attr) {
    LO_CUDA(cudaFuncSetAttribute(attention_fwd_pipe_kernel<T, NVA, NVC, false, ACT, MK>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    LO_CUDA(cudaFuncSetAttribute(attention_fwd_pipe_kernel<T, NVA, NVC, true, ACT, MK>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_MAX));
    attr = true;
  }
  const int ns = att_pipe_splits(x.B, x.nsplit_hint);
  const int rpi = x.rows_per_img > 1 ? x.rows_per_img : 1;
  const int keep_q = att_keep_q((int64_t)(x.B / rpi) * x.R * (C::CHA + C::CHC) * (int64_t)sizeof(T));     // rows of one image: read once
  if (att_grid_cluster((const void*)attention_fwd_pipe_kernel<T, NVA, NVC, false, ACT, MK>, (size_t)C::SMEM, ns, x.B, x.R)) {
    const size_t smem = C::SMEM + (size_t)((x.R + ns - 1) / ns) * 4;
    LO_CUDA(launch_att(attention_fwd_pipe_kernel<T, NVA, NVC, true, ACT, MK>, dim3(ns, x.B), smem, ns, st, att_pdl_ok(x.abi), (const T*)x.att1, (const T*)x.enc,
                       x.att2, x.att2_stride, x.wf, x.alpha, x.alpha_stride, x.ctx, x.gate_pre, x.gate_stride, x.gctx, x.gctx_bf, x.R, ns,
                       (int*)x.work, (float*)((char*)x.work + att_partials_offset(x.B)), keep_q, rpi, x.mask_out));
  } else {
    LO_CUDA(launch_att(attention_fwd_pipe_kernel<T, NVA, NVC, false, ACT, MK>, dim3(ns, x.B), (size_t)C::SMEM, 1, st, att_pdl_ok(x.abi), (const T*)x.att1,
                       (const T*)x.enc, x.att2, x.att2_stride, x.wf, x.alpha, x.alpha_stride, x.ctx, x.gate_pre, x.gate_stride, x.gctx,
                       x.gctx_bf, x.R, ns, (int*)x.work, (float*)((char*)x.work + att_partials_offset(x.B)), keep_q, rpi, x.mask_out));
  }
  LO_LAUNCH_OK();
  return LO_OK;
}

template <typename T, int NVA, int NVC, int ACT>
static int fwd_launch_a(const AttFwdArgs& x, cudaStream_t st) {
  if constexpr (ACT == 0) {
    if (x.mask_out) return fwd_launch_m<T, NVA, NVC, ACT, true>(x, st);        // training: also emit the ReLU mask bits
  }
  return fwd_launch_m<T, NVA, NVC, ACT, false>(x, st);
}

template <typename T, int NVA, int NVC>
static int fwd_launch(const AttFwdArgs& x, cudaStream_t st) {
  return x.act == 1 ? fwd_launch_a<T, NVA, NVC, 1>(x, st) : fwd_launch_a<T, NVA, NVC, 0>(x, st);
}

// C: enc channels; x.a_ch: att1 channels (0 = C).  Supported: A == C in {256, 512, 1024} and (A, C) = (256, 512)
template <typename T>
static int fwd_dispatch(const AttFwdArgs& x, int C, cudaStream_t st) {
  const int A = x.a_ch > 0 ? x.a_ch : C;
  if (A == 256 && C == 512) return fwd_launch<T, 1, 2>(x, st);
  if (A != C) return fail(LO_EINVAL, "%s: attention width pair (%ld, %ld) not instantiated", __func__, A, C);
  if (C == 256) return fwd_launch<T, 1, 1>(x, st);
  if (C == 512) return fwd_launch<T, 2, 2>(x, st);
  return fwd_launch<T, 4, 4>(x, st);
}
int attention_fwd_pipe(const AttFwdArgs& x, int dt, int C, cudaStream_t st) {
  return dt == LO_F32 ? fwd_dispatch<float>(x, C, st) : fwd_dispatch<bf16>(x, C, st);
}

// ---- ragged layout: per-image region counts (decode of images of different sizes)
// rg.map: [B * AP_MAXSPLIT] int4 CTA map, then [B] ticket counters
int64_t attention_ragged_map_bytes(int B) { return (int64_t)B * AP_MAXSPLIT * 16 + (int64_t)B * 4; }

// The split counts follow the dense rule's total: att_pipe_splits(B) per row on average, so equal counts reproduce the dense
// partition and the dense kernel's bits.  Host side: the grid size; device side (one launch per decode call): the map itself.
int attention_ragged_prepare(AttRagged& rg, int B, int rpi, cudaStream_t st) {
  LO_CHECK_ARG(B >= 1 && B <= 6144, "ragged attention: 1 <= rows <= 6144 (shared memory of the map kernel)");
  const int n_img = B / rpi;
  const int ns = att_pipe_splits(B);
  const bool fixed = g_opt_att_nsplit > 0;
  const int64_t sumR = (int64_t)rpi * rg.reg_off_host[n_img];
  int ctas = 0;
  for (int b = 0; b < B; b++)
    ctas += att_ragged_row_splits(ns, B, rg.reg_off_host[b / rpi + 1] - rg.reg_off_host[b / rpi], sumR, fixed);
  rg.ctas = ctas;
  int4* map = (int4*)rg.map;
  attention_ragged_map_kernel<<<1, 512, (size_t)B * 8, st>>>(rg.reg_off, B, rpi, ns, sumR, fixed ? 1 : 0, map,
                                                             (int*)(map + (int64_t)B * AP_MAXSPLIT));
  LO_LAUNCH_OK();
  return LO_OK;
}

template <typename T, int NVA, int NVC, int ACT>
static int fwd_ragged_launch(const AttFwdArgs& x, const AttRagged& rg, cudaStream_t st) {
  using C = ApCfg<T, NVA, NVC>;
  static bool attr = false;
  if (!attr) {
    LO_CUDA(cudaFuncSetAttribute(attention_fwd_ragged_kernel<T, NVA, NVC, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    attr = true;
  }
  const int4* map = (const int4*)rg.map;
  const int rpi = x.rows_per_img > 1 ? x.rows_per_img : 1;
  const int keep_q = att_keep_q((int64_t)rg.reg_off_host[x.B / rpi] * (C::CHA + C::CHC) * (int64_t)sizeof(T));    // all regions, once
  LO_CUDA(launch_att(attention_fwd_ragged_kernel<T, NVA, NVC, ACT>, dim3(rg.ctas), (size_t)C::SMEM, 1, st, true, (const T*)x.att1,
                     (const T*)x.enc, x.att2, x.att2_stride, x.wf, x.alpha, x.alpha_stride, x.ctx, x.gate_pre, x.gate_stride, x.gctx,
                     x.gctx_bf, map, rg.reg_off, rpi, (int*)(map + (int64_t)x.B * AP_MAXSPLIT), (float*)((char*)x.work + att_partials_offset(x.B)), keep_q));
  LO_LAUNCH_OK();
  return LO_OK;
}

template <typename T, int NVA, int NVC>
static int fwd_ragged_act(const AttFwdArgs& x, const AttRagged& rg, cudaStream_t st) {
  return x.act == 1 ? fwd_ragged_launch<T, NVA, NVC, 1>(x, rg, st) : fwd_ragged_launch<T, NVA, NVC, 0>(x, rg, st);
}

// the width pairs of fwd_dispatch: A == C in {256, 512, 1024} with either score, and (A, C) = (256, 512), which only the Genthial
// cell (tanh) uses
template <typename T>
static int fwd_ragged_dispatch(const AttFwdArgs& x, const AttRagged& rg, int C, cudaStream_t st) {
  const int A = x.a_ch > 0 ? x.a_ch : C;
  if (A == 256 && C == 512 && x.act == 1) return fwd_ragged_launch<T, 1, 2, 1>(x, rg, st);
  if (A == C && C == 256) return fwd_ragged_act<T, 1, 1>(x, rg, st);
  if (A == C && C == 512) return fwd_ragged_act<T, 2, 2>(x, rg, st);
  if (A == C && C == 1024) return fwd_ragged_act<T, 4, 4>(x, rg, st);
  return fail(LO_EINVAL, x.act == 1 ? "%s: attention width pair (%ld, %ld), tanh score, not instantiated"
                                    : "%s: attention width pair (%ld, %ld), ReLU score, not instantiated", __func__, A, C);
}
int attention_fwd_ragged(const AttFwdArgs& x, const AttRagged& rg, int dt, int C, cudaStream_t st) {
  return dt == LO_F32 ? fwd_ragged_dispatch<float>(x, rg, C, st) : fwd_ragged_dispatch<bf16>(x, rg, C, st);
}

template <typename T, int NVA, int NVC, int ACT>
static int bwd_launch_a(const AttBwdArgs& x, cudaStream_t st) {
  using C = ApCfg<T, NVA, NVC>;
  static bool attr = false;
  if (!attr) {
    LO_CUDA(cudaFuncSetAttribute(attention_bwd_pipe_kernel<T, NVA, NVC, false, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    LO_CUDA(cudaFuncSetAttribute(attention_bwd_pipe_kernel<T, NVA, NVC, true, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    attr = true;
  }
  const int ns = att_pipe_splits(x.B, x.nsplit_hint);
  if (x.datt1) {
    if constexpr (ACT == 0) {
      LO_CHECK_ARG(!x.mask_in, "d att1 is computed from att1, not from the mask bits");
      static bool attr_d = false;
      if (!attr_d) {
        LO_CUDA(cudaFuncSetAttribute(attention_bwd_pipe_kernel<T, NVA, NVC, false, ACT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
        LO_CUDA(cudaFuncSetAttribute(attention_bwd_pipe_kernel<T, NVA, NVC, true, ACT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
        attr_d = true;
      }
      // without a cluster the splits of a batch row add their d w_full partials with atomics: one split keeps the order fixed
      const int nsd = (x.ordered_dwf && x.dwf_part && !use_cluster(ns, x.R)) ? 1 : ns;
#define LO_BWDD_ARGS                                                                                                             \
  (const T*)x.att1, (const T*)x.enc, x.att2, x.gate, x.o1_stride, x.wf, x.alpha, x.alpha_stride, x.ctx, x.dgctx, x.dg_stride, x.dreg, \
      x.dreg_stride, x.sreg, x.sreg_stride, x.de, x.datt2, x.dgp, x.dcat_stride, x.datt2_bf, x.dgp_bf, x.dctx_out, x.R, nsd,      \
      (int*)x.work, (float*)((char*)x.work + att_partials_offset(x.B)), x.dwf_part, (T*)x.datt1
      if (use_cluster(nsd, x.R)) {
        LO_CUDA(launch_att(attention_bwd_pipe_kernel<T, NVA, NVC, true, ACT, true>, dim3(nsd, x.B), (size_t)C::SMEM, nsd, st, att_pdl_ok(x.abi),
                           LO_BWDD_ARGS));
      } else {
        LO_CUDA(launch_att(attention_bwd_pipe_kernel<T, NVA, NVC, false, ACT, true>, dim3(nsd, x.B), (size_t)C::SMEM, 1, st, att_pdl_ok(x.abi),
                           LO_BWDD_ARGS));
      }
#undef LO_BWDD_ARGS
      LO_LAUNCH_OK();
      return LO_OK;
    }
    return fail(LO_EINVAL, "%s: d att1 is only produced for the ReLU score", __func__);
  }
  if constexpr (ACT == 0 && sizeof(T) == 2 && NVA == 2 && NVC == 2)
  if (x.mask_in && g_opt_att_bwd_mma && att_rows_per_split(x.R, ns) <= 2048) {
    static bool attr_t = false;
    if (!attr_t) {
      LO_CUDA(cudaFuncSetAttribute(attention_bwd_mma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ABM_SMEM + 2048 * 8));
      LO_CUDA(cudaFuncSetAttribute(attention_bwd_mma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ABM_SMEM + 2048 * 8));
      attr_t = true;
    }
#define LO_BWDT_ARGS                                                                                                                  \
  x.mask_in, (const bf16*)x.enc, x.gate, x.o1_stride, x.wf, x.alpha, x.alpha_stride, x.ctx, x.dgctx, x.dg_stride, x.dreg,            \
      x.dreg_stride, x.sreg, x.sreg_stride, x.de, x.datt2, x.dgp, x.dcat_stride, x.datt2_bf, x.dgp_bf, x.dctx_out, x.R, ns,           \
      (int*)x.work, (float*)((char*)x.work + att_partials_offset(x.B)), keep_q, x.att2, x.dwf_part
    // a share of the enc rows kept in L2, the rest evict_first: all 57 MB of enc at cfg #2 do not fit the H100's 50 MB L2, and
    // evict_last on every row was slower than evict_first on every row (47.0 vs 48.1 us per step of the backward loop)
    const int keep_q = att_keep_q((int64_t)x.B * x.R * ABM_CH * 2);
    const size_t smem_t = (size_t)ABM_SMEM + (size_t)att_rows_per_split(x.R, ns) * 8;      // + alpha / d reg of the CTA's rows
    if (att_grid_cluster((const void*)attention_bwd_mma_kernel<false>, smem_t, ns, x.B, x.R)) {
      LO_CUDA(launch_att(attention_bwd_mma_kernel<true>, dim3(ns, x.B), smem_t, ns, st, att_pdl_ok(x.abi), LO_BWDT_ARGS));
    } else {
      LO_CUDA(launch_att(attention_bwd_mma_kernel<false>, dim3(ns, x.B), smem_t, 1, st, att_pdl_ok(x.abi), LO_BWDT_ARGS));
    }
#undef LO_BWDT_ARGS
    LO_LAUNCH_OK();
    return LO_OK;
  }
  if constexpr (ACT == 0) if (x.mask_in) {
    using CM = ApmCfg<T, NVA, NVC>;
    static bool attr_m = false;
    if (!attr_m) {
      LO_CUDA(cudaFuncSetAttribute(attention_bwd_mask_kernel<T, NVA, NVC, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, CM::SMEM));
      LO_CUDA(cudaFuncSetAttribute(attention_bwd_mask_kernel<T, NVA, NVC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, CM::SMEM));
      attr_m = true;
    }
#define LO_BWDM_ARGS                                                                                                                  \
  x.mask_in, (const T*)x.enc, x.gate, x.o1_stride, x.wf, x.alpha, x.alpha_stride, x.ctx, x.dgctx, x.dg_stride, x.dreg, x.dreg_stride, \
      x.sreg, x.sreg_stride, x.de, x.datt2, x.dgp, x.dcat_stride, x.datt2_bf, x.dgp_bf, x.dctx_out, x.R, ns, (int*)x.work,           \
      (float*)((char*)x.work + att_partials_offset(x.B)), x.att2, x.dwf_part
    if (use_cluster(ns, x.R)) {
      LO_CUDA(launch_att(attention_bwd_mask_kernel<T, NVA, NVC, true>, dim3(ns, x.B), (size_t)CM::SMEM, ns, st, att_pdl_ok(x.abi), LO_BWDM_ARGS));
    } else {
      LO_CUDA(launch_att(attention_bwd_mask_kernel<T, NVA, NVC, false>, dim3(ns, x.B), (size_t)CM::SMEM, 1, st, att_pdl_ok(x.abi), LO_BWDM_ARGS));
    }
#undef LO_BWDM_ARGS
    LO_LAUNCH_OK();
    return LO_OK;
  }
#define LO_BWD_ARGS                                                                                                              \
  (const T*)x.att1, (const T*)x.enc, x.att2, x.gate, x.o1_stride, x.wf, x.alpha, x.alpha_stride, x.ctx, x.dgctx, x.dg_stride, x.dreg, \
      x.dreg_stride, x.sreg, x.sreg_stride, x.de, x.datt2, x.dgp, x.dcat_stride, x.datt2_bf, x.dgp_bf, x.dctx_out, x.R, ns,       \
      (int*)x.work, (float*)((char*)x.work + att_partials_offset(x.B)), x.dwf_part, (T*)nullptr
  if (use_cluster(ns, x.R)) {
    LO_CUDA(launch_att(attention_bwd_pipe_kernel<T, NVA, NVC, true, ACT>, dim3(ns, x.B), (size_t)C::SMEM, ns, st, att_pdl_ok(x.abi), LO_BWD_ARGS));
  } else {
    LO_CUDA(launch_att(attention_bwd_pipe_kernel<T, NVA, NVC, false, ACT>, dim3(ns, x.B), (size_t)C::SMEM, 1, st, att_pdl_ok(x.abi), LO_BWD_ARGS));
  }
#undef LO_BWD_ARGS
  LO_LAUNCH_OK();
  return LO_OK;
}

template <typename T, int NVA, int NVC>
static int bwd_launch(const AttBwdArgs& x, cudaStream_t st) {
  return x.act == 1 ? bwd_launch_a<T, NVA, NVC, 1>(x, st) : bwd_launch_a<T, NVA, NVC, 0>(x, st);
}

template <typename T>
static int bwd_dispatch(const AttBwdArgs& x, int C, cudaStream_t st) {
  const int A = x.a_ch > 0 ? x.a_ch : C;
  if (A == 256 && C == 512) return bwd_launch<T, 1, 2>(x, st);
  if (A != C) return fail(LO_EINVAL, "%s: attention width pair (%ld, %ld) not instantiated", __func__, A, C);
  if (C == 256) return bwd_launch<T, 1, 1>(x, st);
  if (C == 512) return bwd_launch<T, 2, 2>(x, st);
  return bwd_launch<T, 4, 4>(x, st);
}
int attention_bwd_pipe(const AttBwdArgs& x, int dt, int C, cudaStream_t st) {
  return dt == LO_F32 ? bwd_dispatch<float>(x, C, st) : bwd_dispatch<bf16>(x, C, st);
}

}  // namespace lo

namespace lo { extern long long* g_tc_dbg; }
extern "C" int lo_debug_buffer(void* p) {
  lo::g_tc_dbg = (long long*)p;
  LO_TRY(lo::cl_set_ts((long long*)p));
  LO_TRY(lo::sk_set_ts((long long*)p));
#ifdef LO_ATT_TIMING
  long long* q = (long long*)p;
  LO_CUDA(cudaMemcpyToSymbol(lo::g_att_ts, &q, sizeof(q)));
#endif
  return LO_OK;
}

// L2 persistence experiment: access-policy window of `stream` over [base, base+bytes) (hit -> persisting, miss -> streaming) and
// the persisting carve-out sized to fit; bytes = 0 resets both.  Attention loads honour it with att_policy_* = 3 (no cache hint).
extern "C" int lo_set_l2_window(const void* base, int64_t bytes, float hit_ratio, void* stream) {
  int dev = 0, max_persist = 0, max_window = 0;
  LO_CUDA(cudaGetDevice(&dev));
  LO_CUDA(cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev));
  LO_CUDA(cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, dev));
  cudaStreamAttrValue v{};
  if (bytes <= 0 || !base) {
    v.accessPolicyWindow.num_bytes = 0;
    lo::g_att_window = v.accessPolicyWindow;
    LO_CUDA(cudaStreamSetAttribute((cudaStream_t)stream, cudaStreamAttributeAccessPolicyWindow, &v));
    LO_CUDA(cudaCtxResetPersistingL2Cache());
    return LO_OK;
  }
  const size_t carve = (size_t)(bytes < max_persist ? bytes : max_persist);
  LO_CUDA(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve));
  v.accessPolicyWindow.base_ptr = const_cast<void*>(base);
  v.accessPolicyWindow.num_bytes = (size_t)(bytes < max_window ? bytes : max_window);
  v.accessPolicyWindow.hitRatio = hit_ratio;
  v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
  v.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
  lo::g_att_window = v.accessPolicyWindow;
  LO_CUDA(cudaStreamSetAttribute((cudaStream_t)stream, cudaStreamAttributeAccessPolicyWindow, &v));
  lo::fail(LO_OK, "l2 window%s: carve %ld B (device max %ld B)", "", (long)carve, (long)max_persist);      // readable via lo_last_error()
  return LO_OK;
}
