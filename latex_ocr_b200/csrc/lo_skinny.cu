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
