// Cluster-fused decoder step kernels: everything between two attention kernels of the time loop in ONE launch whose only
// cross-CTA exchange runs through distributed shared memory of a 16-CTA thread-block cluster.
//
// Why a cluster and not the grid: batch rows are independent in the recurrence (seq2seq_torch.py:304-316), so a block of 16 rows
// (one mma M tile) can be carried through [gates GEMM -> LSTM cell -> next projection] by 16 CTAs that split the OUTPUT columns
// and exchange the 16 x 512 state through DSMEM behind a hardware cluster barrier.  The grid-wide versions
// (dec_step_fwd_kernel / dec_step_bwd_kernel, lo_skinny.cu) needed an all-to-all through L2 — a kernel boundary or a 192-CTA
// atomic barrier, three per direction and step, each costing more than the step's math.  Here 4 clusters (64 rows) x 16 CTAs stream each their 320 KB slice of the weights
// from L2 through a cp.async ring (weights are parameters: the ring is filled before griddepcontrol.wait).
//
// forward  (after attention(t)):   gates = (gate*ctx)_t W_ih[:, E:]^T (+ table row + hh) -> LSTM cell -> h_{t+1}, c_{t+1}
//                                  | cluster barrier, all-gather h_{t+1} |  [att2 | gate_pre | hh]_{t+1} = h_{t+1} W_cat^T + b
// backward (after attention_bwd(t)): dh_t = dh_t(W_hh part) + [datt2 | dgate_pre]_t [W_d ; W_beta] -> LSTM cell backward of step t-1
//                                  | cluster barrier, all-gather dG_{t-1} |  [dgctx | dh]_{t-1} = dG_{t-1} [W_ih[:, E:] | W_hh]
// Same math, same operands (bf16 weights / activations, fp32 accumulation) as the separate kernels; no atomics: every output
// element has one owner, so the backward is bit-reproducible as well.
#include <cooperative_groups.h>

#include "lo_common.cuh"
#include "lo_ptx.cuh"

namespace cg = cooperative_groups;

namespace lo {

constexpr int CLS = 16;           // CTAs per cluster (non-portable size)
constexpr int CL_ROWS = 16;       // batch rows per cluster = one mma M tile
constexpr int CL_THREADS = 256;
constexpr int CL_D = 512;         // decoder_dim = encoder_dim = attention_dim

__device__ __forceinline__ void cl_cp16(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;           // src-size 0 -> zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cl_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cl_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void cl_ldsm4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(saddr));
}
__device__ __forceinline__ void cl_ldsm2(uint32_t& r0, uint32_t& r1, uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(saddr));
}
__device__ __forceinline__ void cl_mma(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cl_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void cl_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cl_wait_bar() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
// 16 bytes from the shared memory of cluster rank `rank` (same offset as `local_saddr` in this CTA)
__device__ __forceinline__ uint4 cl_ld_remote16(uint32_t local_saddr, uint32_t rank) {
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_saddr), "r"(rank));
  uint4 v;
  asm volatile("ld.shared::cluster.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(ra) : "memory");
  return v;
}
__device__ __forceinline__ void cl_st16(uint32_t saddr, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}


// ---- timing build only (-DLO_ATT_TIMING, tools/cl_timeline.py): per-CTA %globaltimer stamps of the last cluster-step launch
#ifdef LO_ATT_TIMING
__device__ long long* g_cl_ts = nullptr;
__device__ __forceinline__ void cl_ts(int k) {
  if (g_cl_ts && threadIdx.x == 0) {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    g_cl_ts[((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * 16 + k] = t;
  }
}
#define CL_TS(k) do { if (ts_on) cl_ts(k); } while (0)
int cl_set_ts(long long* p) { return cudaMemcpyToSymbol(g_cl_ts, &p, sizeof(p)) == cudaSuccess ? LO_OK : LO_ECUDA; }
#else
#define CL_TS(k) do { } while (0)
int cl_set_ts(long long*) { return LO_OK; }
#endif

// ------------------------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int CF_KCH = 64;                          // k elements per weight chunk
constexpr int CF_WPITCH = CF_KCH * 2 + 16;          // 144 B per chunk row: 8 consecutive rows -> 8 different 16-byte bank groups
constexpr int CF_N1 = 4 * CL_D / CLS;               // 128 gate columns per CTA = 32 hidden units x (i, f, g, o)
constexpr int CF_N2 = 6 * CL_D / CLS;               // 192 columns of [att2 | gate_pre | hh] per CTA
constexpr int CF_SLOT = CF_N2 * CF_WPITCH;          // 27 648 B
constexpr int CF_STAGES = 6;
constexpr int CF_APITCH = CL_D * 2 + 16;            // 1040 B per activation row
constexpr int CF_NCH1 = CL_D / CF_KCH;              // 8 chunks per phase
constexpr int CF_OFF_A1 = CF_STAGES * CF_SLOT;
constexpr int CF_OFF_A2 = CF_OFF_A1 + CL_ROWS * CF_APITCH;
constexpr int CF_OFF_H = CF_OFF_A2 + CL_ROWS * CF_APITCH;
constexpr int CF_SMEM = CF_OFF_H + CL_ROWS * (CL_D / CLS) * 2;      // + [16][32] bf16 slab of this CTA's h_{t+1} columns

__global__ void __launch_bounds__(CL_THREADS, 1) dec_cl_fwd_kernel(DecStepFwd p) {
  extern __shared__ __align__(128) uint8_t cl_smem[];
  const uint32_t sbase = smem_u32(cl_smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cr = blockIdx.x;                         // rank in the cluster (cluster = the 16 CTAs of one blockIdx.y)
  const int row0 = blockIdx.y * CL_ROWS;
  const int M = min(CL_ROWS, p.M - row0);            // live rows of this block (>= 1)
  const TcLstmEpi& e = p.e;
  const bool ph2 = p.o1_next != nullptr;
  const int nch = ph2 ? 2 * CF_NCH1 : CF_NCH1;
  const bool ts_on = ph2;           // (timing build) stamp the full launches only
  (void)ts_on;
  CL_TS(0);

  auto issue = [&](int c) {
    if (c < nch) {
      const uint32_t slot = sbase + (uint32_t)(c % CF_STAGES) * CF_SLOT;
      if (c < CF_NCH1) {
        const bf16* w = p.wil + (int64_t)(CF_N1 * cr) * p.ld_wil + c * CF_KCH;
        for (int i = tid; i < CF_N1 * 8; i += CL_THREADS) cl_cp16(slot + (i >> 3) * CF_WPITCH + (i & 7) * 16, w + (int64_t)(i >> 3) * p.ld_wil + (i & 7) * 8, true);
      } else {
        const bf16* w = p.wcat + (int64_t)(CF_N2 * cr) * p.ld_wcat + (c - CF_NCH1) * CF_KCH;
        for (int i = tid; i < CF_N2 * 8; i += CL_THREADS) cl_cp16(slot + (i >> 3) * CF_WPITCH + (i & 7) * 16, w + (int64_t)(i >> 3) * p.ld_wcat + (i & 7) * 8, true);
      }
    }
    cl_commit();
  };
  // weights are parameters: the ring fills before griddepcontrol.wait
#pragma unroll 1
  for (int c = 0; c < CF_STAGES - 1; c++) issue(c);

  // LSTM epilogue operands of this thread's (row, unit) pairs: the table row, the recurrent projection (written by the previous
  // step's launch, two launches back) and c_t do not depend on the preceding attention kernel either
  const int g = lane >> 2, t = lane & 3;
  const bool even = (t & 1) == 0;
  const int row = g + (even ? 0 : 8);
  const bool live = row < M;
  const int D = e.D;
  const int n0 = CF_N1 * cr + 16 * warp;             // first gate column (interleaved: 4 * unit + gate) of this warp
  float add[2][4], cprev[2];
#pragma unroll
  for (int j = 0; j < 2; j++) {
    cprev[j] = 0.f;
#pragma unroll
    for (int q = 0; q < 4; q++) add[j][q] = 0.f;
  }
  if (live) {
    const int64_t gr = row0 + row;
    int64_t tk = e.tok[gr * e.tok_stride];
    if (tk < 0) tk = 0;
    if (tk >= e.V) tk = e.V - 1;
    const float* pt = e.ptab + tk * 4 * D;
    const float* hh = e.hh + gr * e.hh_stride;
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const int u = n0 / 4 + 2 * j + (t >> 1);
      cprev[j] = e.c_prev[gr * D + u];
#pragma unroll
      for (int q = 0; q < 4; q++) add[j][q] = pt[q * D + u] + hh[q * D + u];
    }
  }
  CL_TS(1);
  pdl_wait();
  CL_TS(2);
  pdl_trigger();
  // A of phase 1: (gate * ctx)_t rows of this block (bf16 mirror written by the attention kernel)
  for (int i = tid; i < CL_ROWS * 64; i += CL_THREADS) {
    const int r = i >> 6, sg = i & 63;
    cl_cp16(sbase + CF_OFF_A1 + r * CF_APITCH + sg * 16, p.gctx + (int64_t)(row0 + min(r, M - 1)) * p.ld_gctx + sg * 8, r < M);
  }
  cl_commit();
  cl_wait<0>();
  __syncthreads();
  CL_TS(3);

  float acc1[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  float acc2[3][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  const uint32_t a_lane = (uint32_t)((lane & 7) + ((lane >> 3) & 1) * 8) * CF_APITCH + (uint32_t)(lane >> 4) * 16;
  const uint32_t b_lane = (uint32_t)((lane & 7) + (lane >> 4) * 8) * CF_WPITCH + (uint32_t)((lane >> 3) & 1) * 16;
  const uint32_t b2_lane = (uint32_t)(lane & 7) * CF_WPITCH + (uint32_t)((lane >> 3) & 1) * 16;

  auto lstm_epilogue = [&]() {
    bf16* s_h = reinterpret_cast<bf16*>(cl_smem + CF_OFF_H);
#pragma unroll
    for (int j = 0; j < 2; j++) {
      // even lanes hold (i,f), odd lanes (g,o) of unit u for rows g (acc[.][0..1]) and g+8 (acc[.][2..3])
      const float sx = even ? acc1[j][2] : acc1[j][0], sy = even ? acc1[j][3] : acc1[j][1];
      const float rx = __shfl_xor_sync(0xffffffffu, sx, 1), ry = __shfl_xor_sync(0xffffffffu, sy, 1);
      const int u = n0 / 4 + 2 * j + (t >> 1);
      const int ul = u - (CL_D / CLS) * cr;
      if (!live) {
        s_h[row * (CL_D / CLS) + ul] = __float2bfloat16_rn(0.f);
        continue;
      }
      const float pi = (even ? acc1[j][0] : rx) + add[j][0];
      const float pf = (even ? acc1[j][1] : ry) + add[j][1];
      const float pg = (even ? rx : acc1[j][2]) + add[j][2];
      const float po = (even ? ry : acc1[j][3]) + add[j][3];
      const float ig = sigmoidf_(pi), fg = sigmoidf_(pf), gg = tanhf(pg), og = sigmoidf_(po);
      const float c = fg * cprev[j] + ig * gg;
      const float h = og * tanhf(c);
      const int64_t gr = row0 + row;
      float* gt = e.gates + gr * 4 * D;
      gt[u] = ig; gt[D + u] = fg; gt[2 * D + u] = gg; gt[3 * D + u] = og;
      e.c_out[gr * D + u] = c;
      e.h_out[gr * D + u] = h;
      const bf16 hb = __float2bfloat16_rn(h);
      e.h_bf[gr * D + u] = hb;
      s_h[row * (CL_D / CLS) + ul] = hb;
      if (e.hd) {
        float mult = 1.f;
        if (e.dmask) mult = e.dmask[gr * e.hd_stride + u];
        else if (e.dstate) mult = philox_dropout_mult(e.dstate, e.row0 + (int)gr, e.t_idx, u, e.dp, 1.f / (1.f - e.dp));
        e.hd[gr * e.hd_stride + u] = h * mult;
      }
    }
  };

#pragma unroll 1
  for (int c = 0; c < nch; c++) {
    if (c == CF_NCH1) {
      // ---- phase boundary: LSTM cell, then all-gather h_{t+1} of this row block from the 16 column owners
      CL_TS(4);
      lstm_epilogue();
      CL_TS(9);
      cl_sync_all();
      CL_TS(5);
      for (int i = tid; i < CLS * CL_ROWS * 4; i += CL_THREADS) {
        const int rank = i >> 6, r = (i >> 2) & 15, sg = i & 3;
        const uint4 v = cl_ld_remote16(sbase + CF_OFF_H + r * 64 + sg * 16, (uint32_t)rank);
        cl_st16(sbase + CF_OFF_A2 + r * CF_APITCH + rank * 64 + sg * 16, v);
      }
      CL_TS(6);
      cl_arrive();                                   // peers may exit only after every CTA has read their slab (waited on at the end)
    }
    cl_wait<CF_STAGES - 2>();
    __syncthreads();                                 // chunk c visible to every warp; every warp is done with chunk c-1 (its slot is refilled now)
    issue(c + CF_STAGES - 1);
    const uint32_t slot = sbase + (uint32_t)(c % CF_STAGES) * CF_SLOT;
    if (c < CF_NCH1) {
      const uint32_t ab = sbase + CF_OFF_A1 + a_lane + (uint32_t)c * (CF_KCH * 2);
      const uint32_t bb = slot + (uint32_t)(16 * warp) * CF_WPITCH + b_lane;
#pragma unroll
      for (int kk = 0; kk < CF_KCH / 16; kk++) {
        uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
        cl_ldsm4(a0, a1, a2, a3, ab + kk * 32);
        cl_ldsm4(b0, b1, b2, b3, bb + kk * 32);
        cl_mma(acc1[0], a0, a1, a2, a3, b0, b1);
        cl_mma(acc1[1], a0, a1, a2, a3, b2, b3);
      }
    } else {
      const uint32_t ab = sbase + CF_OFF_A2 + a_lane + (uint32_t)(c - CF_NCH1) * (CF_KCH * 2);
      const uint32_t bb = slot + (uint32_t)(24 * warp) * CF_WPITCH + b_lane;
      const uint32_t bc = slot + (uint32_t)(24 * warp + 16) * CF_WPITCH + b2_lane;
#pragma unroll
      for (int kk = 0; kk < CF_KCH / 16; kk++) {
        uint32_t a0, a1, a2, a3, b0, b1, b2, b3, b4, b5;
        cl_ldsm4(a0, a1, a2, a3, ab + kk * 32);
        cl_ldsm4(b0, b1, b2, b3, bb + kk * 32);
        cl_ldsm2(b4, b5, bc + kk * 32);
        cl_mma(acc2[0], a0, a1, a2, a3, b0, b1);
        cl_mma(acc2[1], a0, a1, a2, a3, b2, b3);
        cl_mma(acc2[2], a0, a1, a2, a3, b4, b5);
      }
    }
  }
  CL_TS(7);
  if (!ph2) {                                        // last step of the sequence: nothing follows the cell
    lstm_epilogue();
    return;
  }
#pragma unroll
  for (int j = 0; j < 3; j++) {
    const int n = CF_N2 * cr + 24 * warp + 8 * j + 2 * t;
    const float bx = p.bcat ? p.bcat[n] : 0.f, by = p.bcat ? p.bcat[n + 1] : 0.f;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int r = g + 8 * h;
      if (r < M) *reinterpret_cast<float2*>(p.o1_next + (int64_t)(row0 + r) * p.ld_o1 + n) = make_float2(acc2[j][2 * h] + bx, acc2[j][2 * h + 1] + by);
    }
  }
  cl_wait_bar();
  CL_TS(8);
}

// ------------------------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int CB_KCH = 128;                         // k elements per weight chunk
constexpr int CB_WPITCH = CB_KCH * 2 + 16;          // 272 B
constexpr int CB_NA = CL_D / CLS;                   // 32 columns of dh per CTA (phase A)
constexpr int CB_NC = 2 * CL_D / CLS;               // 64 columns of [dgctx | dh] per CTA (phase C)
constexpr int CB_KA = 2 * CL_D;                     // K of phase A: A + C = 1024
constexpr int CB_KC = 4 * CL_D;                     // K of phase C: 4D = 2048
constexpr int CB_NCHA = CB_KA / CB_KCH;             // 8
constexpr int CB_NCHC = CB_KC / CB_KCH;             // 16
constexpr int CB_SLOT = CB_NC * CB_WPITCH;          // 17 408 B
constexpr int CB_STAGES = 6;
constexpr int CB_APITCH_A = CB_KA * 2 + 16;         // 2064
constexpr int CB_APITCH_C = CB_KC * 2 + 16;         // 4112
constexpr int CB_OFF_AA = CB_STAGES * CB_SLOT;                       // [16][1024] bf16: datt2 | dgate_pre of step t
constexpr int CB_OFF_AC = CB_OFF_AA + CL_ROWS * CB_APITCH_A;         // [16][2048] bf16: dG of step t-1 (gathered)
constexpr int CB_OFF_DG = CB_OFF_AC + CL_ROWS * CB_APITCH_C;         // [16][4][32] bf16: this CTA's dG columns
constexpr int CB_OFF_RED = CB_OFF_DG + CL_ROWS * 4 * CB_NA * 2;      // [2][16][32] fp32: phase-A partial sums
constexpr int CB_SMEM = CB_OFF_RED + 2 * CL_ROWS * CB_NA * 4;
static_assert(CB_STAGES * CB_SLOT >= 8 * CL_ROWS * CB_NC * 4, "phase-C reduction scratch lives in the ring");

__global__ void __launch_bounds__(CL_THREADS, 1) dec_cl_bwd_kernel(DecStepBwd p) {
  extern __shared__ __align__(128) uint8_t cl_smem[];
  const uint32_t sbase = smem_u32(cl_smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cr = blockIdx.x;
  const int row0 = blockIdx.y * CL_ROWS;
  const bool has_a = p.dcat_a != nullptr, has_bc = p.gates != nullptr;
  const int Ma = has_a ? max(0, min(CL_ROWS, p.Ma - row0)) : 0;      // rows of this block with an attention gradient of step t
  const int Mb = has_bc ? min(CL_ROWS, p.Mb - row0) : min(CL_ROWS, p.Ma - row0);     // rows this launch owns
  const int D = p.D, CD = p.C + p.D;
  const int ncha = has_a ? CB_NCHA : 0;
  const int nch = ncha + (has_bc ? CB_NCHC : 0);
  const bool ts_on = has_a && has_bc;
  (void)ts_on;
  CL_TS(0);

  auto issue = [&](int c) {
    if (c < nch) {
      const uint32_t slot = sbase + (uint32_t)(c % CB_STAGES) * CB_SLOT;
      if (c < ncha) {
        const bf16* w = p.wbwd2 + (int64_t)(CB_NA * cr) * p.ld_w2 + c * CB_KCH;
        for (int i = tid; i < CB_NA * 16; i += CL_THREADS) cl_cp16(slot + (i >> 4) * CB_WPITCH + (i & 15) * 16, w + (int64_t)(i >> 4) * p.ld_w2 + (i & 15) * 8, true);
      } else {
        const bf16* w = p.wbwd1 + (int64_t)(CB_NC * cr) * p.ld_w1 + (c - ncha) * CB_KCH;
        for (int i = tid; i < CB_NC * 16; i += CL_THREADS) cl_cp16(slot + (i >> 4) * CB_WPITCH + (i & 15) * 16, w + (int64_t)(i >> 4) * p.ld_w1 + (i & 15) * 8, true);
      }
    }
    cl_commit();
  };
#pragma unroll 1
  for (int c = 0; c < CB_STAGES - 1; c++) issue(c);

  // LSTM-backward operands of this thread's two (row, unit) pairs: everything but the attention gradient of step t is at least two
  // launches old (gates / cells from the forward pass, dhd from the hoisted fc backward, dc and the W_hh part of dh from the previous
  // launch of this kernel, which the attention kernel in between has waited for)
  const int lr = tid >> 4;                           // block-local row
  const int ul = (tid & 15) * 2;                     // first of two local units
  const int u = CB_NA * cr + ul;
  const int64_t gr = row0 + lr;
  const bool live = lr < Mb;
  float gi[2], gf[2], gg[2], go[2], tc[2], cpv[2], dhd[2], dcv[2], dhb[2];
#pragma unroll
  for (int k = 0; k < 2; k++) { gi[k] = gf[k] = gg[k] = go[k] = tc[k] = cpv[k] = dhd[k] = dcv[k] = dhb[k] = 0.f; }
  if (live) {
    const float2 b2 = *reinterpret_cast<const float2*>(p.dxh + gr * CD + p.C + u);
    dhb[0] = b2.x; dhb[1] = b2.y;
    if (has_bc) {
      const float* gt = p.gates + gr * 4 * D;
      const float2 x0 = *reinterpret_cast<const float2*>(gt + u), x1 = *reinterpret_cast<const float2*>(gt + D + u);
      const float2 x2 = *reinterpret_cast<const float2*>(gt + 2 * D + u), x3 = *reinterpret_cast<const float2*>(gt + 3 * D + u);
      const float2 cc = *reinterpret_cast<const float2*>(p.c_cur + gr * D + u), cp = *reinterpret_cast<const float2*>(p.c_prev + gr * D + u);
      const float2 dd = *reinterpret_cast<const float2*>(p.dhd + gr * p.dhd_stride + u), dc2 = *reinterpret_cast<const float2*>(p.dc + gr * D + u);
      gi[0] = x0.x; gi[1] = x0.y; gf[0] = x1.x; gf[1] = x1.y; gg[0] = x2.x; gg[1] = x2.y; go[0] = x3.x; go[1] = x3.y;
      tc[0] = tanhf(cc.x); tc[1] = tanhf(cc.y); cpv[0] = cp.x; cpv[1] = cp.y; dhd[0] = dd.x; dhd[1] = dd.y; dcv[0] = dc2.x; dcv[1] = dc2.y;
      float m0 = 1.f, m1 = 1.f;
      if (p.dmask) {
        const float2 mm = *reinterpret_cast<const float2*>(p.dmask + gr * p.dhd_stride + u);
        m0 = mm.x; m1 = mm.y;
      } else if (p.dstate) {
        m0 = philox_dropout_mult(p.dstate, (int)gr, p.t_idx, u, p.dp, 1.f / (1.f - p.dp));
        m1 = philox_dropout_mult(p.dstate, (int)gr, p.t_idx, u + 1, p.dp, 1.f / (1.f - p.dp));
      }
      dhd[0] *= m0; dhd[1] *= m1;
    }
  }
  CL_TS(1);
  pdl_wait();
  CL_TS(2);
  pdl_trigger();
  if (has_a) {
    for (int i = tid; i < CL_ROWS * 128; i += CL_THREADS) {
      const int r = i >> 7, sg = i & 127;
      cl_cp16(sbase + CB_OFF_AA + r * CB_APITCH_A + sg * 16, p.dcat_a + (int64_t)(row0 + min(r, max(Ma, 1) - 1)) * p.ld_dcat + sg * 8, r < Ma);
    }
  }
  cl_commit();
  cl_wait<0>();
  __syncthreads();
  CL_TS(3);

  const int g = lane >> 2, t = lane & 3;
  const uint32_t a_lane_a = (uint32_t)((lane & 7) + ((lane >> 3) & 1) * 8) * CB_APITCH_A + (uint32_t)(lane >> 4) * 16;
  const uint32_t a_lane_c = (uint32_t)((lane & 7) + ((lane >> 3) & 1) * 8) * CB_APITCH_C + (uint32_t)(lane >> 4) * 16;
  float accA[4] = {0.f, 0.f, 0.f, 0.f};
  float accC[8][4];
#pragma unroll
  for (int j = 0; j < 8; j++)
#pragma unroll
    for (int q = 0; q < 4; q++) accC[j][q] = 0.f;

  // dh of this thread's pairs after phase A
  float dh[2] = {dhb[0], dhb[1]};

  auto lstm_bwd_and_gather = [&]() {
    // ---- phase A results: the two K halves meet in shared memory
    if (has_a) {
      float* red = reinterpret_cast<float*>(cl_smem + CB_OFF_RED) + (warp >> 2) * (CL_ROWS * CB_NA);
      const int nt = warp & 3;
      red[g * CB_NA + nt * 8 + 2 * t] = accA[0];
      red[g * CB_NA + nt * 8 + 2 * t + 1] = accA[1];
      red[(g + 8) * CB_NA + nt * 8 + 2 * t] = accA[2];
      red[(g + 8) * CB_NA + nt * 8 + 2 * t + 1] = accA[3];
      __syncthreads();
      const float* r0p = reinterpret_cast<const float*>(cl_smem + CB_OFF_RED);
      dh[0] += r0p[lr * CB_NA + ul] + r0p[CL_ROWS * CB_NA + lr * CB_NA + ul];
      dh[1] += r0p[lr * CB_NA + ul + 1] + r0p[CL_ROWS * CB_NA + lr * CB_NA + ul + 1];
    }
    if (!has_bc) {                                   // last launch of the loop: dh_0 only
      if (live) *reinterpret_cast<float2*>(p.dxh + gr * CD + p.C + u) = make_float2(dh[0], dh[1]);
      return;
    }
    // ---- LSTM cell backward of step t-1 (seq2seq_torch.py:313 autograd), two units per thread
    __nv_bfloat162* s_dg = reinterpret_cast<__nv_bfloat162*>(cl_smem + CB_OFF_DG);     // [16][4][16] pairs
    float v[4][2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const float dht = dhd[k] + dh[k];
      const float dct = dcv[k] + dht * go[k] * (1.f - tc[k] * tc[k]);
      v[0][k] = dct * gg[k] * gi[k] * (1.f - gi[k]);
      v[1][k] = dct * cpv[k] * gf[k] * (1.f - gf[k]);
      v[2][k] = dct * gi[k] * (1.f - gg[k] * gg[k]);
      v[3][k] = dht * tc[k] * go[k] * (1.f - go[k]);
      dcv[k] = dct * gf[k];
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
      __nv_bfloat162 b;
      b.x = __float2bfloat16_rn(live ? v[q][0] : 0.f);
      b.y = __float2bfloat16_rn(live ? v[q][1] : 0.f);
      s_dg[(lr * 4 + q) * (CB_NA / 2) + (ul >> 1)] = b;
      if (live) {
        *reinterpret_cast<float2*>(p.dG + gr * p.dG_stride + q * D + u) = make_float2(v[q][0], v[q][1]);
        *reinterpret_cast<__nv_bfloat162*>(p.dG_bf + gr * p.dG_stride + q * D + u) = b;
      }
    }
    if (live) *reinterpret_cast<float2*>(p.dc + gr * D + u) = make_float2(dcv[0], dcv[1]);
    CL_TS(9);
    cl_sync_all();
    CL_TS(5);
    // all-gather dG_{t-1} of this row block: [16][4 gates][16 ranks x 32 units]
    for (int i = tid; i < CLS * CL_ROWS * 4 * 4; i += CL_THREADS) {
      const int rank = i >> 8, r = (i >> 4) & 15, q = (i >> 2) & 3, sg = i & 3;
      const uint4 x = cl_ld_remote16(sbase + CB_OFF_DG + (r * 4 + q) * (CB_NA * 2) + sg * 16, (uint32_t)rank);
      cl_st16(sbase + CB_OFF_AC + r * CB_APITCH_C + (q * CL_D + rank * CB_NA) * 2 + sg * 16, x);
    }
    CL_TS(6);
    cl_arrive();
  };

  if (!has_a && has_bc) lstm_bwd_and_gather();       // first launch of the loop: no attention gradient yet
#pragma unroll 1
  for (int c = 0; c < nch; c++) {
    if (has_a && c == ncha) { CL_TS(4); lstm_bwd_and_gather(); }   // (only reached when phase C follows)
    cl_wait<CB_STAGES - 2>();
    __syncthreads();
    issue(c + CB_STAGES - 1);
    const uint32_t slot = sbase + (uint32_t)(c % CB_STAGES) * CB_SLOT;
    if (c < ncha) {
      // phase A: warp = (n tile of 8 columns, half of the chunk's 8 k-steps)
      const int nt = warp & 3, kh = warp >> 2;
      const uint32_t ab = sbase + CB_OFF_AA + a_lane_a + (uint32_t)c * (CB_KCH * 2) + (uint32_t)kh * 128;
      const uint32_t bb = slot + (uint32_t)(nt * 8 + (lane & 7)) * CB_WPITCH + (uint32_t)(lane >> 3) * 16 + (uint32_t)kh * 128;
#pragma unroll
      for (int kp = 0; kp < 2; kp++) {
        uint32_t b0, b1, b2, b3, a0, a1, a2, a3;
        cl_ldsm4(b0, b1, b2, b3, bb + kp * 64);      // 8 columns x 32 k: (b0, b1) first k-step, (b2, b3) second
        cl_ldsm4(a0, a1, a2, a3, ab + kp * 64);
        cl_mma(accA, a0, a1, a2, a3, b0, b1);
        cl_ldsm4(a0, a1, a2, a3, ab + kp * 64 + 32);
        cl_mma(accA, a0, a1, a2, a3, b2, b3);
      }
    } else {
      // phase C: warp = one of the chunk's 8 k-steps, all 64 columns
      const uint32_t ab = sbase + CB_OFF_AC + a_lane_c + (uint32_t)(c - ncha) * (CB_KCH * 2) + (uint32_t)warp * 32;
      const uint32_t bb = slot + (uint32_t)((lane & 7) + (lane >> 4) * 8) * CB_WPITCH + (uint32_t)((lane >> 3) & 1) * 16 + (uint32_t)warp * 32;
      uint32_t a0, a1, a2, a3;
      cl_ldsm4(a0, a1, a2, a3, ab);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        uint32_t b0, b1, b2, b3;
        cl_ldsm4(b0, b1, b2, b3, bb + (uint32_t)(16 * j) * CB_WPITCH);
        cl_mma(accC[2 * j], a0, a1, a2, a3, b0, b1);
        cl_mma(accC[2 * j + 1], a0, a1, a2, a3, b2, b3);
      }
    }
  }
  if (!has_bc) {
    lstm_bwd_and_gather();
    return;
  }
  CL_TS(7);
  // ---- phase C results: the 8 k-step owners meet in shared memory (the ring is free: every chunk has been consumed)
  __syncthreads();
  float* red = reinterpret_cast<float*>(cl_smem);                      // [8][16][64]
#pragma unroll
  for (int j = 0; j < 8; j++) {
    float* o = red + warp * (CL_ROWS * CB_NC);
    o[g * CB_NC + j * 8 + 2 * t] = accC[j][0];
    o[g * CB_NC + j * 8 + 2 * t + 1] = accC[j][1];
    o[(g + 8) * CB_NC + j * 8 + 2 * t] = accC[j][2];
    o[(g + 8) * CB_NC + j * 8 + 2 * t + 1] = accC[j][3];
  }
  __syncthreads();
  {
    const int r = tid >> 4, n4 = (tid & 15) * 4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int w = 0; w < 8; w++) {
      const float4 x = *reinterpret_cast<const float4*>(red + w * (CL_ROWS * CB_NC) + r * CB_NC + n4);
      s.x += x.x; s.y += x.y; s.z += x.z; s.w += x.w;
    }
    if (r < Mb) *reinterpret_cast<float4*>(p.dxh + (int64_t)(row0 + r) * CD + CB_NC * cr + n4) = s;
  }
  cl_wait_bar();
  CL_TS(8);
}

// ------------------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------------------
template <typename P>
static cudaError_t launch_cluster(void (*kernel)(P), int row_blocks, size_t smem, cudaStream_t st, const P& p) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(CLS, row_blocks);
  cfg.blockDim = dim3(CL_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CLS;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = g_opt_pdl ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, p);
}

// 1 = 16-CTA clusters of these kernels can be scheduled on this device, 0 = not (the callers fall back to the separate launches)
template <typename P>
static int cluster_ready(void (*kernel)(P), size_t smem, int* state) {
  if (*state >= 0) return *state;
  *state = 0;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
      cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(CLS, 4);
  cfg.blockDim = dim3(CL_THREADS);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CLS;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  *state = n >= 1 ? 1 : 0;
  return *state;
}

static int g_cl_fwd_state = -1, g_cl_bwd_state = -1;

bool dec_cl_fwd_ok(int D, int C, int N2) {
  return g_opt_dec_cl && D == CL_D && C == CL_D && N2 == CLS * CF_N2 && cluster_ready(dec_cl_fwd_kernel, CF_SMEM, &g_cl_fwd_state);
}
bool dec_cl_bwd_ok(int D, int C, int A) {
  return g_opt_dec_cl_bwd && D == CL_D && C == CL_D && A == CL_D && cluster_ready(dec_cl_bwd_kernel, CB_SMEM, &g_cl_bwd_state);
}

int dec_cl_fwd(const DecStepFwd& p, cudaStream_t st) {
  LO_CHECK_ARG(p.M >= 1 && p.K == CL_D && p.e.D == CL_D && p.N2 == CLS * CF_N2 && p.e.h_bf, "cluster step: D = C = 512, O1 = 3072");
  LO_CHECK_ARG(p.ld_gctx % 8 == 0 && p.ld_wil % 8 == 0 && p.ld_wcat % 8 == 0 && p.ld_o1 % 2 == 0, "16-byte aligned rows");
  LO_CUDA(launch_cluster(dec_cl_fwd_kernel, cdiv(p.M, CL_ROWS), (size_t)CF_SMEM, st, p));
  LO_LAUNCH_OK();
  return LO_OK;
}

int dec_cl_bwd(const DecStepBwd& p, cudaStream_t st) {
  LO_CHECK_ARG(p.D == CL_D && p.C == CL_D && p.K2 == CB_KA && p.K1 == CB_KC, "cluster step: D = C = A = 512");
  LO_CHECK_ARG(p.dcat_a != nullptr || p.gates != nullptr, "nothing to do");
  LO_CHECK_ARG(p.ld_dcat % 8 == 0 && p.ld_w1 % 8 == 0 && p.ld_w2 % 8 == 0 && p.dG_stride % 8 == 0 && p.dhd_stride % 2 == 0, "aligned rows");
  const int rows = p.gates ? p.Mb : p.Ma;
  LO_CHECK_ARG(rows >= 1, "row count");
  LO_CUDA(launch_cluster(dec_cl_bwd_kernel, cdiv(rows, CL_ROWS), (size_t)CB_SMEM, st, p));
  LO_LAUNCH_OK();
  return LO_OK;
}

}  // namespace lo
