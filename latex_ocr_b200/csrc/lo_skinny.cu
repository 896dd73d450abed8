// Latency-optimised GEMM for the decoder's per-step projections: C[M <= 64][N] (+)= A[M][K] * W[N][K]^T + bias.
//
// These GEMMs are 33-134 MFLOP with M = batch = 64 rows: nothing about them is throughput bound.  The wgmma path
// (lo_tc.cu, kept and selectable with lo_set_option("skinny_mma", 0)) pays a fixed pipeline latency per launch
// (barrier setup, a TMA round trip per K block, the accumulator epilogue).  Here
// every CTA (16 output columns x all 64 rows x one K slice) issues ALL of its loads at once with cp.async (one L2
// round trip), then runs warp-level mma.sync from shared memory and stores straight from the accumulator registers.
// The FLOP-heavy work (convolutions, att1, weight gradients, logits) stays on wgmma.
#include "lo_common.cuh"
#include "lo_ptx.cuh"

namespace lo {

constexpr int SK_KC = 512;        // K elements per CTA
constexpr int SK_NT = 16;         // output columns per CTA
constexpr int SK_PITCH = SK_KC + 8;   // bf16 elements per smem row (+16 B: conflict-free ldmatrix)
constexpr int SK_SMEM = (64 + SK_NT) * SK_PITCH * 2;

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;           // src-size 0 -> zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma_bf16_16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// grid (N/16, ksplit, row blocks of 64), 128 threads (warp w owns rows 16w..16w+15 of its row block)
// TMA = true: both operands arrive as 1-D bulk copies (cp.async.bulk, one per row, issued by warp 0, completion on two mbarriers)
// instead of 16-byte cp.async, which moves the post-wait 64 KB activation load through one SM's LDGSTS path far more slowly.
template <bool TMA>
__global__ void __launch_bounds__(128) skinny_mma_kernel(const bf16* __restrict__ A, int64_t lda, const bf16* __restrict__ W, int64_t ldw,
                                                          float* __restrict__ C, int64_t ldc, int M, int N, int K, int kc,
                                                          const float* __restrict__ bias, int mode) {
  A += (int64_t)blockIdx.z * 64 * lda;
  C += (int64_t)blockIdx.z * 64 * ldc;
  M = min(64, M - (int)blockIdx.z * 64);
  extern __shared__ __align__(16) uint8_t sk_smem[];
  bf16* sA = reinterpret_cast<bf16*>(sk_smem);               // [64][SK_PITCH]
  bf16* sW = sA + 64 * SK_PITCH;                             // [16][SK_PITCH]
  const int n0 = blockIdx.x * SK_NT;
  const int k0 = blockIdx.y * kc;
  const int kn = min(kc, K - k0);                            // multiple of 16
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cpr = kn / 8;                                    // 16-byte chunks per row
  // the bias is a parameter: fetched up front instead of after the MMA loop (one L2 round trip off the tail of the launch)
  float bpre[2][2];
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const int n = n0 + j * 8 + 2 * (lane & 3);
    const bool has = bias && blockIdx.y == 0 && n < N;
    bpre[j][0] = has ? bias[n] : 0.f;
    bpre[j][1] = has ? bias[n + 1] : 0.f;
  }
  if constexpr (TMA) {
    uint64_t* bars = reinterpret_cast<uint64_t*>(sk_smem + SK_SMEM);      // [0] weights, [1] activations
    if (tid == 0) {
      mbar_init(bars, 1);
      mbar_init(bars + 1, 1);
      fence_barrier_init();
    }
    __syncthreads();
    const uint32_t row_bytes = (uint32_t)kn * 2u;
    if (warp == 0) {
      // PDL: the weight slice never depends on the preceding launch -> fetched before griddepcontrol.wait
      const int wrows = min(SK_NT, N - n0);
      const uint64_t pol = l2_policy_evict_last();
      if (lane == 0) mbar_expect_tx(bars, (uint32_t)wrows * row_bytes);
      __syncwarp();
      if (lane < wrows) bulk_g2s(sW + lane * SK_PITCH, W + (int64_t)(n0 + lane) * ldw + k0, row_bytes, bars, pol);
    }
    // rows the copies do not write are zero (cp.async zero-fill semantics of the other path)
    for (int i = tid; i < (SK_NT - min(SK_NT, N - n0)) * cpr; i += 128)
      *reinterpret_cast<uint4*>(sW + (min(SK_NT, N - n0) + i / cpr) * SK_PITCH + (i % cpr) * 8) = make_uint4(0, 0, 0, 0);
    for (int i = tid; i < (64 - M) * cpr; i += 128)
      *reinterpret_cast<uint4*>(sA + (M + i / cpr) * SK_PITCH + (i % cpr) * 8) = make_uint4(0, 0, 0, 0);
    pdl_wait();
    pdl_trigger();
    if (warp == 0) {
      const uint64_t pol = l2_policy_evict_first();
      if (lane == 0) mbar_expect_tx(bars + 1, (uint32_t)M * row_bytes);
      __syncwarp();
      for (int r = lane; r < M; r += 32) bulk_g2s(sA + r * SK_PITCH, A + (int64_t)r * lda + k0, row_bytes, bars + 1, pol);
    }
    mbar_wait(bars, 0);
    mbar_wait(bars + 1, 0);
    __syncthreads();                                         // the zero-filled rows
  } else {
  // PDL: the weight slice never depends on the preceding launch -> fetch it before griddepcontrol.wait
  for (int i = tid; i < SK_NT * cpr; i += 128) {
    const int r = i / cpr, c = i % cpr;
    cp_async16(sW + r * SK_PITCH + c * 8, W + (int64_t)min(n0 + r, N - 1) * ldw + k0 + c * 8, n0 + r < N);
  }
  pdl_wait();
  pdl_trigger();
  for (int i = tid; i < 64 * cpr; i += 128) {
    const int r = i / cpr, c = i % cpr;
    cp_async16(sA + r * SK_PITCH + c * 8, A + (int64_t)min(r, M - 1) * lda + k0 + c * 8, r < M);
  }
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  }
  // two independent accumulator sets (even / odd k-steps): the 32-step chain of dependent mma.sync per warp was a visible part of
  // these latency-bound launches (4 warps per CTA, ~1.3 CTAs per SM: nothing else hides it)
  float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  float acd[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  const bf16* a_ptr = sA + (warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * SK_PITCH + (lane >> 4) * 8;
  const bf16* b_ptr = sW + ((lane & 7) + (lane >> 4) * 8) * SK_PITCH + ((lane >> 3) & 1) * 8;
  int k = 0;
#pragma unroll 4
  for (; k + 32 <= kn; k += 32) {
    uint32_t a0, a1, a2, a3, b0, b1, b2, b3, c0, c1, c2, c3, d0, d1, d2, d3;
    ldmatrix_x4(a0, a1, a2, a3, a_ptr + k);
    ldmatrix_x4(b0, b1, b2, b3, b_ptr + k);
    ldmatrix_x4(c0, c1, c2, c3, a_ptr + k + 16);
    ldmatrix_x4(d0, d1, d2, d3, b_ptr + k + 16);
    mma_bf16_16816(acc[0], a0, a1, a2, a3, b0, b1);          // columns n0 .. n0+7
    mma_bf16_16816(acc[1], a0, a1, a2, a3, b2, b3);          // columns n0+8 .. n0+15
    mma_bf16_16816(acd[0], c0, c1, c2, c3, d0, d1);
    mma_bf16_16816(acd[1], c0, c1, c2, c3, d2, d3);
  }
  if (k < kn) {
    uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
    ldmatrix_x4(a0, a1, a2, a3, a_ptr + k);
    ldmatrix_x4(b0, b1, b2, b3, b_ptr + k);
    mma_bf16_16816(acc[0], a0, a1, a2, a3, b0, b1);
    mma_bf16_16816(acc[1], a0, a1, a2, a3, b2, b3);
  }
#pragma unroll
  for (int j = 0; j < 2; j++)
#pragma unroll
    for (int q = 0; q < 4; q++) acc[j][q] += acd[j][q] + bpre[j][q & 1];
  if (gridDim.y > 1 && mode != 1) {
    // ordered split K: the K slices of this tile are one cluster; rank 0 (slice 0) adds the partials in slice order, alone writes C
    __syncthreads();                                         // every ldmatrix read of sA is done: it stages the partials
    float* part = reinterpret_cast<float*>(sk_smem);
#pragma unroll
    for (int i = 0; i < 8; i++) part[i * 128 + tid] = acc[i >> 2][i & 3];
    cl_sync();
    if (cl_rank() == 0) {
      float s[8];
      cl_sum_n<8>(part + tid, 128, s);
#pragma unroll
      for (int i = 0; i < 8; i++) acc[i >> 2][i & 3] = s[i];
    }
    cl_sync();
    if (cl_rank() != 0) return;
  }
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const int n = n0 + j * 8 + 2 * t;
    if (n >= N) continue;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int r = warp * 16 + g + h * 8;
      if (r >= M) continue;
      float* o = C + (int64_t)r * ldc + n;
      float x = acc[j][2 * h], y = acc[j][2 * h + 1];
      if (mode == 1) {
        atomicAdd(o, x);
        atomicAdd(o + 1, y);
        continue;
      }
      if (mode == 2) { const float2 old = *reinterpret_cast<float2*>(o); x += old.x; y += old.y; }
      *reinterpret_cast<float2*>(o) = make_float2(x, y);
    }
  }
}

// The same GEMM over the gate-interleaved context half of weight_ih (row 4*u + gate, lo_decoder.cu:interleave_wih_kernel) with the
// LSTM cell (nn.LSTMCell, gates i,f,g,o: seq2seq_torch.py:313) in the epilogue: a CTA's 16 columns are 4 whole hidden units, lane
// pairs (t, t^1) hold (i,f) and (g,o) of one unit for rows g and g+8 and swap halves with one shuffle, so every thread finalises
// one (row, unit).  The table row, the recurrent projection and c_{t-1} are fetched BEFORE the MMA loop (they do not depend on
// it), which a separate GEMM epilogue could not hide.  K <= 512 (one slice).  Replaces gemm + lstm_pw_fwd_kernel.
__global__ void __launch_bounds__(128) skinny_lstm_kernel(const bf16* __restrict__ A, int64_t lda, const bf16* __restrict__ Wil, int64_t ldw,
                                                           int M, int K, TcLstmEpi e) {
  extern __shared__ __align__(16) uint8_t sk_smem[];
  bf16* sA = reinterpret_cast<bf16*>(sk_smem);
  bf16* sW = sA + 64 * SK_PITCH;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sk_smem + SK_SMEM);      // [0] weights, [1] activations
  const int n0 = blockIdx.x * SK_NT;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cpr = K / 8;
  const uint32_t row_bytes = (uint32_t)K * 2u;
  if (tid == 0) {
    mbar_init(bars, 1);
    mbar_init(bars + 1, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (warp == 0) {                         // weights: a parameter, bulk copies issued before griddepcontrol.wait
    const uint64_t pol = l2_policy_evict_last();
    if (lane == 0) mbar_expect_tx(bars, (uint32_t)SK_NT * row_bytes);
    __syncwarp();
    if (lane < SK_NT) bulk_g2s(sW + lane * SK_PITCH, Wil + (int64_t)(n0 + lane) * ldw, row_bytes, bars, pol);
  }
  for (int i = tid; i < (64 - M) * cpr; i += 128)
    *reinterpret_cast<uint4*>(sA + (M + i / cpr) * SK_PITCH + (i % cpr) * 8) = make_uint4(0, 0, 0, 0);
  // epilogue operands of this thread's (row, unit) pairs.  The token's table row, the recurrent projection of THIS step (written by the
  // projection kernel two launches back: the attention kernel in between has waited for it) and c_t are all older than the preceding
  // launch: fetched before griddepcontrol.wait, so the two dependent round trips (token, then its table row) leave the critical path
  const int D = e.D;
  const int g = lane >> 2, t = lane & 3;
  const bool even = (t & 1) == 0;
  const int row = warp * 16 + g + (even ? 0 : 8);
  const bool live = row < M;
  float add[2][4], cprev[2];
#pragma unroll
  for (int j = 0; j < 2; j++) {
    cprev[j] = 0.f;
#pragma unroll
    for (int q = 0; q < 4; q++) add[j][q] = 0.f;
  }
  if (live) {
    int64_t tk = e.tok[(int64_t)row * e.tok_stride];
    if (tk < 0) tk = 0;
    if (tk >= e.V) tk = e.V - 1;
    const float* pt = e.ptab + tk * 4 * D;
    const float* hh = e.hh + (int64_t)row * e.hh_stride;
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const int u = n0 / 4 + 2 * j + (t >> 1);
      cprev[j] = e.c_prev[(int64_t)row * D + u];
#pragma unroll
      for (int q = 0; q < 4; q++) add[j][q] = pt[q * D + u] + hh[q * D + u];
    }
  }
  pdl_wait();
  pdl_trigger();
  if (warp == 0) {
    const uint64_t pol = l2_policy_evict_first();
    if (lane == 0) mbar_expect_tx(bars + 1, (uint32_t)M * row_bytes);
    __syncwarp();
    for (int r = lane; r < M; r += 32) bulk_g2s(sA + r * SK_PITCH, A + (int64_t)r * lda, row_bytes, bars + 1, pol);
  }
  mbar_wait(bars, 0);
  mbar_wait(bars + 1, 0);
  __syncthreads();                         // the zero-filled rows
  float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  const bf16* a_ptr = sA + (warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * SK_PITCH + (lane >> 4) * 8;
  const bf16* b_ptr = sW + ((lane & 7) + (lane >> 4) * 8) * SK_PITCH + ((lane >> 3) & 1) * 8;
#pragma unroll 4
  for (int k = 0; k < K; k += 16) {
    uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
    ldmatrix_x4(a0, a1, a2, a3, a_ptr + k);
    ldmatrix_x4(b0, b1, b2, b3, b_ptr + k);
    mma_bf16_16816(acc[0], a0, a1, a2, a3, b0, b1);
    mma_bf16_16816(acc[1], a0, a1, a2, a3, b2, b3);
  }
#pragma unroll
  for (int j = 0; j < 2; j++) {
    // even lanes hold (i,f), odd lanes (g,o) of unit u for rows g (acc[.][0..1]) and g+8 (acc[.][2..3])
    const float sx = even ? acc[j][2] : acc[j][0], sy = even ? acc[j][3] : acc[j][1];
    const float rx = __shfl_xor_sync(0xffffffffu, sx, 1), ry = __shfl_xor_sync(0xffffffffu, sy, 1);
    if (!live) continue;
    const float pi = (even ? acc[j][0] : rx) + add[j][0];
    const float pf = (even ? acc[j][1] : ry) + add[j][1];
    const float pg = (even ? rx : acc[j][2]) + add[j][2];
    const float po = (even ? ry : acc[j][3]) + add[j][3];
    const int u = n0 / 4 + 2 * j + (t >> 1);
    const float ig = sigmoidf_(pi), fg = sigmoidf_(pf), gg = tanhf(pg), og = sigmoidf_(po);
    const float c = fg * cprev[j] + ig * gg;
    const float h = og * tanhf(c);
    float* gt = e.gates + (int64_t)row * 4 * D;
    gt[u] = ig; gt[D + u] = fg; gt[2 * D + u] = gg; gt[3 * D + u] = og;
    e.c_out[(int64_t)row * D + u] = c;
    e.h_out[(int64_t)row * D + u] = h;
    if (e.h_bf) e.h_bf[(int64_t)row * D + u] = __float2bfloat16_rn(h);
    if (e.hd) {
      float mult = 1.f;
      if (e.dmask) mult = e.dmask[(int64_t)row * e.hd_stride + u];
      else if (e.dstate) mult = philox_dropout_mult(e.dstate, e.row0 + row, e.t_idx, u, e.dp, 1.f / (1.f - e.dp));
      e.hd[(int64_t)row * e.hd_stride + u] = h * mult;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------------------
// Fused decoder forward step: one launch per time step instead of three.
//   phase 1 (CTAs 0 .. 4D/16-1): gates = (gate*ctx)_t W_ih[:, E:]^T with the LSTM cell in the epilogue -> h_{t+1}, c_{t+1}
//   grid barrier (all CTAs are co-resident: <= 2 per SM by shared memory, grid <= 2 x LO_NUM_SMS)
//   phase 2 (CTAs 0 .. N2/16-1): [att2 | gate_pre | hh_pre]_{t+1} = h_{t+1} [W_d; W_beta; W_hh]^T + b
// The time loop is a chain of dependent 64-row GEMMs: each separate launch costs several times its math in pure
// latency (launch, cold loads, drain).  Here both weight slices are fetched before griddepcontrol.wait, the barrier costs one L2 atomic
// round trip, and h_{t+1} is re-read from L2 where the other CTAs just put it.  griddepcontrol.launch_dependents is issued only
// AFTER the barrier: by then every CTA of this grid is resident, so the early-starting attention kernel of the next step
// cannot take a slot a not-yet-resident CTA of this grid needs (no deadlock).
// ------------------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Arrival counters are spread over GB_NC cache lines (one L2 atomic unit each): a CTA adds 1 to counter (blockIdx.x % GB_NC) with a
// fire-and-forget red.release, warp 0 polls all GB_NC counters with ONE acquire load per lane and sums them with a warp reduce.  Arrivals
// on a single counter serialise in the L2 atomic unit (as much as a kernel boundary for a full grid); spread over GB_NC counters
// they cost a small fraction of that.  Counters are monotonic: `target` is the
// total number of arrivals after this barrier.
constexpr int GB_NC = 16;
__device__ __forceinline__ void grid_barrier(unsigned int* ctr, unsigned int target) {
  __syncthreads();
  if (threadIdx.x < 32) {
    if (threadIdx.x == 0)
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr + (blockIdx.x % GB_NC) * 32) : "memory");
    const long long t0 = clock64();
    while (true) {
      unsigned int v = threadIdx.x < GB_NC ? ld_acquire_u32(ctr + threadIdx.x * 32) : 0u;
      v = __reduce_add_sync(0xffffffffu, v);
      if (v >= target) break;
      if (clock64() - t0 > 4000000000LL) __trap();          // a protocol bug must fail loudly, not hang the GPU
    }
  }
  __syncthreads();
}


// ---- timing build only (-DLO_ATT_TIMING, tools/fuse_timeline.py): per-CTA %globaltimer stamps of the last fused-step launch
#ifdef LO_ATT_TIMING
__device__ long long* g_sk_ts = nullptr;
__device__ __forceinline__ void sk_ts(int k) {
  if (g_sk_ts && threadIdx.x == 0) {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    g_sk_ts[(int64_t)blockIdx.x * 16 + k] = t;
  }
}
#define SK_TS(k) do { if (ts_on) sk_ts(k); } while (0)
int sk_set_ts(long long* p) { return cudaMemcpyToSymbol(g_sk_ts, &p, sizeof(p)) == cudaSuccess ? LO_OK : LO_ECUDA; }
#else
#define SK_TS(k) do { } while (0)
int sk_set_ts(long long*) { return LO_OK; }
#endif

constexpr int SKF_SMEM = (64 + 2 * SK_NT) * SK_PITCH * 2;

__global__ void __launch_bounds__(128) dec_step_fwd_kernel(DecStepFwd p) {
  extern __shared__ __align__(16) uint8_t sk_smem[];
  bf16* sA = reinterpret_cast<bf16*>(sk_smem);               // [64][SK_PITCH]   A of phase 1, then of phase 2
  bf16* sW1 = sA + 64 * SK_PITCH;                            // [16][SK_PITCH]   Wil slice
  bf16* sW2 = sW1 + SK_NT * SK_PITCH;                        // [16][SK_PITCH]   Wcat slice
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.x * SK_NT;
  const int K = p.K, cpr = K / 8, M = p.M;
  const TcLstmEpi& e = p.e;
  const bool ph1 = n0 < 4 * e.D;
  const bool ph2 = p.o1_next != nullptr && n0 < p.N2;
  const bool ts_on = p.o1_next != nullptr;
  (void)ts_on;
  SK_TS(0);
  // ---- weights of both phases: parameters, independent of the preceding launches
  if (ph1)
    for (int i = tid; i < SK_NT * cpr; i += 128) {
      const int r = i / cpr, c = i % cpr;
      cp_async16(sW1 + r * SK_PITCH + c * 8, p.wil + (int64_t)(n0 + r) * p.ld_wil + c * 8, true);
    }
  if (ph2)
    for (int i = tid; i < SK_NT * cpr; i += 128) {
      const int r = i / cpr, c = i % cpr;
      cp_async16(sW2 + r * SK_PITCH + c * 8, p.wcat + (int64_t)min(n0 + r, p.N2 - 1) * p.ld_wcat + c * 8, n0 + r < p.N2);
    }
  // the LSTM epilogue's operands (token -> table row, recurrent projection of THIS step, c_t) were all written at least two launches
  // back (the attention kernel in between has waited for them): fetched before griddepcontrol.wait, two dependent L2 round trips
  // (token, then its table row) leave the critical path
  const int g = lane >> 2, t = lane & 3;
  const int D = e.D;
  const bool even = (t & 1) == 0;
  const int row = warp * 16 + g + (even ? 0 : 8);
  const bool live = row < M;
  float add[2][4], cprev[2];
#pragma unroll
  for (int j = 0; j < 2; j++) {
    cprev[j] = 0.f;
#pragma unroll
    for (int q = 0; q < 4; q++) add[j][q] = 0.f;
  }
  if (ph1 && live) {
    int64_t tk = e.tok[(int64_t)row * e.tok_stride];
    if (tk < 0) tk = 0;
    if (tk >= e.V) tk = e.V - 1;
    const float* pt = e.ptab + tk * 4 * D;
    const float* hh = e.hh + (int64_t)row * e.hh_stride;
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const int u = n0 / 4 + 2 * j + (t >> 1);
      cprev[j] = e.c_prev[(int64_t)row * D + u];
#pragma unroll
      for (int q = 0; q < 4; q++) add[j][q] = pt[q * D + u] + hh[q * D + u];
    }
  }
  SK_TS(1);
  pdl_wait();
  SK_TS(2);
  const bf16* a_ptr = sA + (warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * SK_PITCH + (lane >> 4) * 8;
  if (ph1) {
    for (int i = tid; i < 64 * cpr; i += 128) {
      const int r = i / cpr, c = i % cpr;
      cp_async16(sA + r * SK_PITCH + c * 8, p.gctx + (int64_t)min(r, M - 1) * p.ld_gctx + c * 8, r < M);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    SK_TS(3);
    float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    const bf16* b_ptr = sW1 + ((lane & 7) + (lane >> 4) * 8) * SK_PITCH + ((lane >> 3) & 1) * 8;
#pragma unroll 4
    for (int k = 0; k < K; k += 16) {
      uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
      ldmatrix_x4(a0, a1, a2, a3, a_ptr + k);
      ldmatrix_x4(b0, b1, b2, b3, b_ptr + k);
      mma_bf16_16816(acc[0], a0, a1, a2, a3, b0, b1);
      mma_bf16_16816(acc[1], a0, a1, a2, a3, b2, b3);
    }
#pragma unroll
    for (int j = 0; j < 2; j++) {
      // even lanes hold (i,f), odd lanes (g,o) of unit u for rows g (acc[.][0..1]) and g+8 (acc[.][2..3])
      const float sx = even ? acc[j][2] : acc[j][0], sy = even ? acc[j][3] : acc[j][1];
      const float rx = __shfl_xor_sync(0xffffffffu, sx, 1), ry = __shfl_xor_sync(0xffffffffu, sy, 1);
      if (!live) continue;
      const float pi = (even ? acc[j][0] : rx) + add[j][0];
      const float pf = (even ? acc[j][1] : ry) + add[j][1];
      const float pg = (even ? rx : acc[j][2]) + add[j][2];
      const float po = (even ? ry : acc[j][3]) + add[j][3];
      const int u = n0 / 4 + 2 * j + (t >> 1);
      const float ig = sigmoidf_(pi), fg = sigmoidf_(pf), gg = tanhf(pg), og = sigmoidf_(po);
      const float c = fg * cprev[j] + ig * gg;
      const float h = og * tanhf(c);
      float* gt = e.gates + (int64_t)row * 4 * D;
      gt[u] = ig; gt[D + u] = fg; gt[2 * D + u] = gg; gt[3 * D + u] = og;
      e.c_out[(int64_t)row * D + u] = c;
      e.h_out[(int64_t)row * D + u] = h;
      e.h_bf[(int64_t)row * D + u] = __float2bfloat16_rn(h);
      if (e.hd) {
        float mult = 1.f;
        if (e.dmask) mult = e.dmask[(int64_t)row * e.hd_stride + u];
        else if (e.dstate) mult = philox_dropout_mult(e.dstate, e.row0 + row, e.t_idx, u, e.dp, 1.f / (1.f - e.dp));
        e.hd[(int64_t)row * e.hd_stride + u] = h * mult;
      }
    }
  } else {
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  if (p.o1_next == nullptr) {             // last step: nothing follows the cell
    pdl_trigger();
    return;
  }
  SK_TS(4);
  grid_barrier(p.bar, p.bar_target);       // h_{t+1} of every CTA is in L2 (also orders this CTA's reads of sA before reuse)
  SK_TS(5);
  pdl_trigger();
  if (!ph2) return;
  for (int i = tid; i < 64 * cpr; i += 128) {
    const int r = i / cpr, c = i % cpr;
    cp_async16(sA + r * SK_PITCH + c * 8, e.h_bf + (int64_t)min(r, M - 1) * e.D + c * 8, r < M);     // cp.async.cg: from L2
  }
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  SK_TS(6);
  float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  const bf16* b_ptr = sW2 + ((lane & 7) + (lane >> 4) * 8) * SK_PITCH + ((lane >> 3) & 1) * 8;
#pragma unroll 4
  for (int k = 0; k < K; k += 16) {
    uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
    ldmatrix_x4(a0, a1, a2, a3, a_ptr + k);
    ldmatrix_x4(b0, b1, b2, b3, b_ptr + k);
    mma_bf16_16816(acc[0], a0, a1, a2, a3, b0, b1);
    mma_bf16_16816(acc[1], a0, a1, a2, a3, b2, b3);
  }
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const int n = n0 + j * 8 + 2 * t;
    if (n >= p.N2) continue;
    const float bx = p.bcat ? p.bcat[n] : 0.f, by = p.bcat ? p.bcat[n + 1] : 0.f;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int r = warp * 16 + g + h * 8;
      if (r >= M) continue;
      *reinterpret_cast<float2*>(p.o1_next + (int64_t)r * p.ld_o1 + n) = make_float2(acc[j][2 * h] + bx, acc[j][2 * h + 1] + by);
    }
  }
  SK_TS(7);
}

int dec_step_fwd(const DecStepFwd& p, cudaStream_t st) {
  LO_CHECK_ARG(p.M >= 1 && p.M <= 64 && p.K % 16 == 0 && p.K <= SK_KC && p.e.D == p.K && p.e.D % 4 == 0 && p.N2 % 2 == 0, "M<=64, K=D<=512");
  LO_CHECK_ARG(p.e.h_bf && p.bar, "bf16 mirror of h and the barrier counter are required");
  static bool attr = false;
  if (!attr) {
    LO_CUDA(cudaFuncSetAttribute(dec_step_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SKF_SMEM));
    attr = true;
  }
  const int n1 = 4 * p.e.D / SK_NT, n2 = p.o1_next ? cdiv(p.N2, SK_NT) : 0;
  const int grid = n1 > n2 ? n1 : n2;
  LO_CHECK_ARG(grid <= 296, "fused step: grid must be co-resident (<= 2 CTAs per SM)");
  LO_CUDA(launch_pdl(dec_step_fwd_kernel, dim3(grid), dim3(128), (size_t)SKF_SMEM, st, p));
  LO_LAUNCH_OK();
  return LO_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// Fused decoder backward step (see DecStepBwd): one launch instead of three between two attention-backward kernels.
// grid = (C+D)/16 column tiles x 4 K slices of phase C = 256 CTAs (co-resident: 2 per SM); phase A uses the first D/16 x 2.
// ------------------------------------------------------------------------------------------------------------------------------
// one 64 x 16 x kn tile: C[r][n0 + ..] += sum_k A[r][k0 + k] W[n0 + ..][k0 + k]   (fp32 atomics)
__device__ __forceinline__ void skinny_tile_atomic(const bf16* sA, const bf16* sW, int kn, float* C, int64_t ldc, int n0, int N, int M) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  const bf16* a_ptr = sA + (warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * SK_PITCH + (lane >> 4) * 8;
  const bf16* b_ptr = sW + ((lane & 7) + (lane >> 4) * 8) * SK_PITCH + ((lane >> 3) & 1) * 8;
#pragma unroll 4
  for (int k = 0; k < kn; k += 16) {
    uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
    ldmatrix_x4(a0, a1, a2, a3, a_ptr + k);
    ldmatrix_x4(b0, b1, b2, b3, b_ptr + k);
    mma_bf16_16816(acc[0], a0, a1, a2, a3, b0, b1);
    mma_bf16_16816(acc[1], a0, a1, a2, a3, b2, b3);
  }
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const int n = n0 + j * 8 + 2 * t;
    if (n >= N) continue;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int r = warp * 16 + g + h * 8;
      if (r >= M) continue;
      float* o = C + (int64_t)r * ldc + n;
      atomicAdd(o, acc[j][2 * h]);
      atomicAdd(o + 1, acc[j][2 * h + 1]);
    }
  }
}

__global__ void __launch_bounds__(128) dec_step_bwd_kernel(DecStepBwd p) {
  extern __shared__ __align__(16) uint8_t sk_smem[];
  bf16* sA = reinterpret_cast<bf16*>(sk_smem);               // [64][SK_PITCH]
  bf16* sWa = sA + 64 * SK_PITCH;                            // [16][SK_PITCH]  wbwd2 slice (phase A)
  bf16* sWc = sWa + SK_NT * SK_PITCH;                        // [16][SK_PITCH]  wbwd1 slice (phase C)
  const int tid = threadIdx.x;
  const int cta = blockIdx.x;
  const int D = p.D, CD = p.C + p.D;
  // roles
  const int na_tiles = D / SK_NT, ka_slices = p.K2 / SK_KC;            // phase A: na_tiles x ka_slices CTAs
  const bool has_a = p.dcat_a != nullptr && cta < na_tiles * ka_slices;
  const int a_n0 = (cta % na_tiles) * SK_NT, a_k0 = (cta / na_tiles) * SK_KC;
  const int nc_tiles = CD / SK_NT;                                     // phase C: nc_tiles x (K1 / 512) CTAs = the whole grid
  const bool has_bc = p.gates != nullptr;
  const int c_n0 = (cta % nc_tiles) * SK_NT, c_k0 = (cta / nc_tiles) * SK_KC;
  const bool has_c = has_bc && c_k0 < p.K1;
  constexpr int cpr = SK_KC / 8;
  // ---- weight slices: parameters, fetched before griddepcontrol.wait
  if (has_a)
    for (int i = tid; i < SK_NT * cpr; i += 128) {
      const int r = i / cpr, c = i % cpr;
      cp_async16(sWa + r * SK_PITCH + c * 8, p.wbwd2 + (int64_t)(a_n0 + r) * p.ld_w2 + a_k0 + c * 8, true);
    }
  if (has_c)
    for (int i = tid; i < SK_NT * cpr; i += 128) {
      const int r = i / cpr, c = i % cpr;
      cp_async16(sWc + r * SK_PITCH + c * 8, p.wbwd1 + (int64_t)(c_n0 + r) * p.ld_w1 + c_k0 + c * 8, true);
    }
  pdl_wait();
  unsigned int target = p.bar_target;
  if (p.dcat_a != nullptr) {
    if (has_a) {
      for (int i = tid; i < 64 * cpr; i += 128) {
        const int r = i / cpr, c = i % cpr;
        cp_async16(sA + r * SK_PITCH + c * 8, p.dcat_a + (int64_t)min(r, p.Ma - 1) * p.ld_dcat + a_k0 + c * 8, r < p.Ma);
      }
      asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
      __syncthreads();
      skinny_tile_atomic(sA, sWa, SK_KC, p.dxh + p.C, CD, a_n0, D, p.Ma);
    }
    if (!has_bc) {                           // last launch of the loop: only the projection back to dh_0
      pdl_trigger();
      return;
    }
    grid_barrier(p.bar, target);             // dh_{t-1} complete
    target += gridDim.x;
  }
  // ---- phase B: LSTM cell backward of step t-1, one (row, unit) per thread over the whole grid
  {
    const int total = p.Mb * D;
    for (int idx = cta * 128 + tid; idx < total; idx += gridDim.x * 128) {
      const int b = idx / D, j = idx % D;
      const float* gt = p.gates + (int64_t)b * 4 * D;
      const float i = gt[j], f = gt[D + j], g = gt[2 * D + j], o = gt[3 * D + j];
      const float tc = tanhf(p.c_cur[(int64_t)b * D + j]);
      float dh = p.dhd[(int64_t)b * p.dhd_stride + j];
      if (p.dmask) dh *= p.dmask[(int64_t)b * p.dhd_stride + j];
      else if (p.dstate) dh *= philox_dropout_mult(p.dstate, b, p.t_idx, j, p.dp, 1.f / (1.f - p.dp));
      float* z = p.dxh + (int64_t)b * CD;
      dh += __ldcg(z + p.C + j);                               // written by other CTAs' atomics (L2)
      const float dct = p.dc[(int64_t)b * D + j] + dh * o * (1.f - tc * tc);
      float v[4];
      v[0] = dct * g * i * (1.f - i);
      v[1] = dct * p.c_prev[(int64_t)b * D + j] * f * (1.f - f);
      v[2] = dct * i * (1.f - g * g);
      v[3] = dh * tc * o * (1.f - o);
      p.dc[(int64_t)b * D + j] = dct * f;
      float* d = p.dG + (int64_t)b * p.dG_stride;
      bf16* q = p.dG_bf + (int64_t)b * p.dG_stride;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        d[k * D + j] = v[k];
        q[k * D + j] = __float2bfloat16_rn(v[k]);
      }
      // clear [dgctx | dh] for the atomics of phase C (dh_next was consumed above; C == D so column j covers the dgctx half)
      z[p.C + j] = 0.f;
      for (int c = j; c < p.C; c += D) z[c] = 0.f;
    }
  }
  grid_barrier(p.bar, target);               // dG_{t-1} (bf16 mirror) of every row is in L2, dxh is cleared
  pdl_trigger();
  if (!has_c) return;
  for (int i = tid; i < 64 * cpr; i += 128) {
    const int r = i / cpr, c = i % cpr;
    cp_async16(sA + r * SK_PITCH + c * 8, p.dG_bf + (int64_t)min(r, p.Mb - 1) * p.dG_stride + c_k0 + c * 8, r < p.Mb);
  }
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  skinny_tile_atomic(sA, sWc, SK_KC, p.dxh, CD, c_n0, CD, p.Mb);
}

int dec_step_bwd(const DecStepBwd& p, cudaStream_t st) {
  LO_CHECK_ARG(p.K2 % SK_KC == 0 && p.K1 % SK_KC == 0 && p.D % SK_NT == 0 && (p.C + p.D) % SK_NT == 0 && p.C == p.D, "K1, K2 multiples of 512, C == D");
  LO_CHECK_ARG((p.dcat_a == nullptr || (p.Ma >= 1 && p.Ma <= 64)) && (p.gates == nullptr || (p.Mb >= 1 && p.Mb <= 64)), "row counts <= 64");
  LO_CHECK_ARG(p.bar && p.dxh, "null pointer");
  static bool attr = false;
  if (!attr) {
    LO_CUDA(cudaFuncSetAttribute(dec_step_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SKF_SMEM));
    attr = true;
  }
  const int grid = ((p.C + p.D) / SK_NT) * (p.K1 / SK_KC);
  LO_CHECK_ARG(grid <= 296 && grid >= (p.D / SK_NT) * (p.K2 / SK_KC), "fused step: grid must be co-resident and cover phase A");
  LO_CUDA(launch_pdl(dec_step_bwd_kernel, dim3(grid), dim3(128), (size_t)SKF_SMEM, st, p));
  LO_LAUNCH_OK();
  return LO_OK;
}

int skinny_gemm_nt_lstm(const bf16* A, int64_t lda, const bf16* Wil, int64_t ldw, int M, int D, int K, const TcLstmEpi& e, cudaStream_t st) {
  LO_CHECK_ARG(M >= 1 && M <= 64 && K % 16 == 0 && K <= SK_KC && lda % 8 == 0 && ldw % 8 == 0 && D % 4 == 0, "M<=64, K%16, K<=512");
  static bool attr = false;
  if (!attr) {
    LO_CUDA(cudaFuncSetAttribute(skinny_lstm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_SMEM + 16));
    attr = true;
  }
  LO_CUDA(launch_pdl(skinny_lstm_kernel, dim3(4 * D / SK_NT), dim3(128), (size_t)SK_SMEM + 16, st, A, lda, Wil, ldw, M, K, e));
  LO_LAUNCH_OK();
  return LO_OK;
}

// atomic_acc: the product is added onto C (C holds the base values).  splits > 1: the K slices add their partial sums onto C with
// fp32 atomics, or — option "deterministic" — groups of up to 8 slices run as one thread-block cluster each, summed in slice order
// and added onto C group after group in stream order (run-to-run identical results)
int skinny_gemm_nt(const bf16* A, int64_t lda, const bf16* W, int64_t ldw, float* C, int64_t ldc, int M, int N, int K, const float* bias,
                   int splits, int atomic_acc, cudaStream_t st) {
  LO_CHECK_ARG(M >= 1 && M <= 64 * 1024 && K % 16 == 0 && N % 2 == 0 && lda % 8 == 0 && ldw % 8 == 0 && ldc % 2 == 0, "K%16, ld%8");
  static bool attr = false;
  if (!attr) {
    LO_CUDA(cudaFuncSetAttribute(skinny_mma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_SMEM));
    LO_CUDA(cudaFuncSetAttribute(skinny_mma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_SMEM + 16));
    attr = true;
  }
  int ks = cdiv(K, SK_KC);
  if (splits > ks) ks = splits;
  int kc = cdiv(cdiv(K, ks), 16) * 16;
  if (kc > SK_KC) kc = SK_KC;
  ks = cdiv(K, kc);
  if (!g_opt_det || ks == 1) {
    const int mode = (ks > 1 || atomic_acc) ? 1 : 0;
    if (ks > 1 && !atomic_acc) LO_CUDA(cudaMemset2DAsync(C, (size_t)ldc * 4, 0, (size_t)N * 4, (size_t)M, st));
    const dim3 grid(cdiv(N, SK_NT), ks, cdiv(M, 64));
    if (g_opt_skinny_tma) {
      LO_CUDA(launch_pdl(skinny_mma_kernel<true>, grid, dim3(128), (size_t)SK_SMEM + 16, st, A, lda, W, ldw, C, ldc, M, N, K, kc, bias, mode));
    } else {
      LO_CUDA(launch_pdl(skinny_mma_kernel<false>, grid, dim3(128), (size_t)SK_SMEM, st, A, lda, W, ldw, C, ldc, M, N, K, kc, bias, mode));
    }
    LO_LAUNCH_OK();
    return LO_OK;
  }
  for (int k0 = 0; k0 < K; k0 += 8 * kc) {
    const int kg = K - k0 < 8 * kc ? K - k0 : 8 * kc, ng = cdiv(kg, kc);
    const int mode = (k0 > 0 || atomic_acc) ? 2 : 0;
    const float* bg = k0 == 0 ? bias : nullptr;
    const dim3 grid(cdiv(N, SK_NT), ng, cdiv(M, 64)), cl(1, ng, 1);
    if (g_opt_skinny_tma) {
      LO_CUDA(launch_cluster(skinny_mma_kernel<true>, grid, dim3(128), (size_t)SK_SMEM + 16, st, cl, true, A + k0, lda, W + k0, ldw, C, ldc, M,
                             N, kg, kc, bg, mode));
    } else {
      LO_CUDA(launch_cluster(skinny_mma_kernel<false>, grid, dim3(128), (size_t)SK_SMEM, st, cl, true, A + k0, lda, W + k0, ldw, C, ldc, M, N,
                             kg, kc, bg, mode));
    }
    LO_LAUNCH_OK();
  }
  return LO_OK;
}

}  // namespace lo
