// CUDA-core (SIMT) strided batched GEMM with fp32 accumulation — the tight-parity path and the
// fallback for shapes the wgmma kernels (lo_tc.cu) do not take.  Replaces the torch.mm / nn.Linear
// library calls behind seq2seq_torch.py:172-176, :223-227 (and their autograd twins).
#include "lo_common.cuh"
#include "lo_ptx.cuh"

namespace lo {

char g_err[512] = "";
int64_t g_launches = 0;

template <typename TA, typename TB, typename TC, int BM, int BN, int BK, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
gemm_simt_kernel(const TA* __restrict__ A, const TB* __restrict__ B, TC* __restrict__ C, GemmDesc d, int splitk) {
  constexpr int NT = (BM / TM) * (BN / TN);
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int bz = blockIdx.z / splitk, sk = blockIdx.z % splitk;
  A += (int64_t)bz * d.sA;
  B += (int64_t)bz * d.sB;
  C += (int64_t)bz * d.sC;
  // K range of this split (multiples of BK)
  const int kchunks = (d.K + BK - 1) / BK;
  const int cps = (kchunks + splitk - 1) / splitk;
  const int kbeg = sk * cps * BK;
  const int kend = min(d.K, (sk + 1) * cps * BK);
  const bool a_kfast = (d.sak == 1), b_kfast = (d.sbk == 1);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; i++)
#pragma unroll
    for (int j = 0; j < TN; j++) acc[i][j] = 0.f;

  for (int k0 = kbeg; k0 < kend; k0 += BK) {
    for (int i = tid; i < BM * BK; i += NT) {
      int m, k;
      if (a_kfast) { k = i % BK; m = i / BK; } else { m = i % BM; k = i / BM; }
      float v = 0.f;
      if (m0 + m < d.M && k0 + k < kend) v = ldf(A + (int64_t)(m0 + m) * d.sam + (int64_t)(k0 + k) * d.sak);
      As[k][m] = v;
    }
    for (int i = tid; i < BN * BK; i += NT) {
      int n, k;
      if (b_kfast) { k = i % BK; n = i / BK; } else { n = i % BN; k = i / BN; }
      float v = 0.f;
      if (n0 + n < d.N && k0 + k < kend) v = ldf(B + (int64_t)(k0 + k) * d.sbk + (int64_t)(n0 + n) * d.sbn);
      Bs[k][n] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; k++) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i++) a[i] = As[k][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; j++) b[j] = Bs[k][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; i++) {
    const int m = m0 + ty * TM + i;
    if (m >= d.M) continue;
#pragma unroll
    for (int j = 0; j < TN; j++) {
      const int n = n0 + tx * TN + j;
      if (n >= d.N) continue;
      float v = acc[i][j];
      TC* cp = C + (int64_t)m * d.ldc + n;
      if (splitk > 1) {
        if (sk == 0 && d.bias) v += d.bias[n];
        if constexpr (sizeof(TC) == 4) atomicAdd(reinterpret_cast<float*>(cp), v);
      } else {
        if (d.bias) v += d.bias[n];
        if (d.accumulate) v += ldf(cp);
        if (d.relu) v = fmaxf(v, 0.f);
        stf(cp, v);
      }
    }
  }
}

template <typename TA, typename TB, typename TC>
static int launch_simt(const TA* A, const TB* B, TC* C, const GemmDesc& d, int splitk, cudaStream_t st) {
  const long tiles64 = (long)cdiv(d.M, 64) * cdiv(d.N, 64) * d.batch * splitk;
  if (tiles64 >= 120 || (d.M > 64 && d.N > 64 && tiles64 >= 64)) {
    dim3 grid(cdiv(d.N, 64), cdiv(d.M, 64), d.batch * splitk);
    gemm_simt_kernel<TA, TB, TC, 64, 64, 16, 4, 4><<<grid, 256, 0, st>>>(A, B, C, d, splitk);
  } else {
    dim3 grid(cdiv(d.N, 32), cdiv(d.M, 32), d.batch * splitk);
    gemm_simt_kernel<TA, TB, TC, 32, 32, 16, 2, 2><<<grid, 256, 0, st>>>(A, B, C, d, splitk);
  }
  LO_LAUNCH_OK();
  return LO_OK;
}

__global__ void zero2d_kernel(float* C, int M, int N, int64_t ldc, int64_t sC) {
  float* c = C + (int64_t)blockIdx.z * sC;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (int64_t)M * N; i += (int64_t)gridDim.x * blockDim.x)
    c[(i / N) * ldc + (i % N)] = 0.f;
}

int gemm(const void* A, int dtA, const void* B, int dtB, void* C, int dtC, const GemmDesc& d, int impl, cudaStream_t st) {
  LO_CHECK_ARG(d.M > 0 && d.N > 0 && d.K > 0 && d.batch > 0, "empty GEMM");
  if (impl == LO_IMPL_TC && dtA == LO_BF16 && dtB == LO_BF16 && d.sak == 1 && d.sbk == 1 && d.batch == 1 && d.sam % 8 == 0 &&
      d.sbn % 8 == 0 && tc_available()) {
    // few rows, fp32 result: the latency-optimised mma.sync kernel (lo_skinny.cu) — same path as the decoder's per-step GEMMs;
    // up to 512 rows (row blocks of 64) when the shape does not qualify for wgmma (e.g. beam-search logits with V % 8 != 0)
    const bool tc_ok = d.K % 64 == 0 && d.N % 8 == 0 && d.ldc % 8 == 0;
    if (g_opt_skinny_mma && (d.M <= 64 || (!tc_ok && d.M <= 512)) && dtC == LO_F32 && !d.relu && d.K % 16 == 0 && d.N % 2 == 0 &&
        d.ldc % 2 == 0)
      return skinny_gemm_nt((const bf16*)A, d.sam, (const bf16*)B, d.sbn, (float*)C, d.ldc, d.M, d.N, d.K, d.bias, 1, d.accumulate, st);
    // otherwise wgmma; few rows -> 64-wide N tiles (twice the CTAs)
    if (tc_ok)
      return tc_gemm_nt_ex((const bf16*)A, d.sam, (const bf16*)B, d.sbn, C, dtC, d.ldc, d.M, d.N, d.K, d.bias, d.accumulate, d.relu, 1, 0,
                           d.M <= 64 ? 1 : 0, st);
  }
  // C = A^T B with both operands stored [K][.] (weight gradients): wgmma MN-major kernel, split-K atomics onto a cleared C
  if (impl == LO_IMPL_TC && dtA == LO_BF16 && dtB == LO_BF16 && dtC == LO_F32 && d.sam == 1 && d.sbn == 1 && d.batch == 1 && !d.bias &&
      !d.relu && !d.accumulate && d.sak % 8 == 0 && d.sbk % 8 == 0 && d.M >= 64 && d.N >= 64 && ((uintptr_t)A & 15) == 0 &&
      ((uintptr_t)B & 15) == 0 && tc_available()) {
    LO_CUDA(cudaMemset2DAsync(C, (size_t)d.ldc * 4, 0, (size_t)d.N * 4, (size_t)d.M, st));
    return tc_gemm_tn((const bf16*)A, d.sak, (const bf16*)B, d.sbk, (float*)C, d.ldc, d.M, d.N, d.K, st);
  }
  // split-K only for fp32 outputs without ReLU when the tile grid would leave most SMs idle and K is long.  Option
  // "deterministic": at most two splits, onto a zeroed C only — two addends onto 0 sum the same in either order
  int splitk = 1;
  if (dtC == LO_F32 && !d.relu && d.K >= 2048 && !(g_opt_det && d.accumulate)) {
    const long tiles = (long)cdiv(d.M, 64) * cdiv(d.N, 64) * d.batch;
    if (tiles < 2 * LO_NUM_SMS) {
      splitk = (int)((2 * LO_NUM_SMS + tiles - 1) / tiles);
      const int maxs = g_opt_det ? 2 : d.K / 256;
      if (splitk > maxs) splitk = maxs;
      if (splitk < 1) splitk = 1;
    }
  }
  GemmDesc dd = d;
  if (splitk > 1) {
    if (!d.accumulate) {
      zero2d_kernel<<<dim3(cdiv((long)d.M * d.N, 1024), 1, d.batch), 256, 0, st>>>((float*)C, d.M, d.N, d.ldc, d.sC);
      LO_LAUNCH_OK();
    }
    dd.accumulate = 1;
  }
#define LO_GEMM_CASE(a, b, c, TA_, TB_, TC_) \
  if (dtA == a && dtB == b && dtC == c) return launch_simt<TA_, TB_, TC_>((const TA_*)A, (const TB_*)B, (TC_*)C, dd, splitk, st);
  LO_GEMM_CASE(LO_F32, LO_F32, LO_F32, float, float, float)
  LO_GEMM_CASE(LO_F32, LO_BF16, LO_F32, float, bf16, float)
  LO_GEMM_CASE(LO_BF16, LO_BF16, LO_BF16, bf16, bf16, bf16)
  LO_GEMM_CASE(LO_BF16, LO_BF16, LO_F32, bf16, bf16, float)
  LO_GEMM_CASE(LO_BF16, LO_F32, LO_F32, bf16, float, float)
  LO_GEMM_CASE(LO_F32, LO_F32, LO_BF16, float, float, bf16)
#undef LO_GEMM_CASE
  return fail(LO_EINVAL, "lo_gemm: unsupported dtype combination%s (%ld,%ld)", "", dtA * 10 + dtB, dtC);
}

int gemm_nt(const void* A, int dtA, int64_t lda, const void* W, int dtW, int64_t ldw, void* C, int dtC, int64_t ldc,
            int M, int N, int K, const float* bias, int accumulate, int relu, int impl, cudaStream_t st) {
  GemmDesc d{M, N, K, lda, 1, 1, ldw, ldc, 1, 0, 0, 0, bias, accumulate, relu};
  return gemm(A, dtA, W, dtW, C, dtC, d, impl, st);
}
int gemm_tn(const void* A, int dtA, int64_t lda, const void* B, int dtB, int64_t ldb, void* C, int dtC, int64_t ldc,
            int M, int N, int K, int accumulate, int impl, cudaStream_t st) {
  GemmDesc d{M, N, K, 1, lda, ldb, 1, ldc, 1, 0, 0, 0, nullptr, accumulate, 0};
  return gemm(A, dtA, B, dtB, C, dtC, d, impl, st);
}
int gemm_nn(const void* A, int dtA, int64_t lda, const void* B, int dtB, int64_t ldb, void* C, int dtC, int64_t ldc,
            int M, int N, int K, int accumulate, int impl, cudaStream_t st) {
  GemmDesc d{M, N, K, lda, 1, ldb, 1, ldc, 1, 0, 0, 0, nullptr, accumulate, 0};
  return gemm(A, dtA, B, dtB, C, dtC, d, impl, st);
}

// out[n] (+)= sum_m X[m][n]: every row split of a column block adds its partial sums with one fp32 atomic per column.  Option
// "deterministic": the row splits of a column block form one thread-block cluster whose rank 0 adds their partial sums in rank
// order (lo_ptx.cuh:cl_sum); without `accumulate` up to two clusters cover a column block and add onto the zeroed `out` with one
// fp32 atomic each — two addends onto 0 give the same sum in either order.  Without a cluster launch the kernels' cluster is
// the block itself.
constexpr int CS_MAXCL = 16;          // non-portable cluster size (H100)
constexpr int CS_THREADS = 1024;

// a warp reads 256 consecutive columns of one row (8 per lane, 16 B for bf16), the block's 32 warps stride the rows, 4 rows in flight
template <typename T>
__global__ void __launch_bounds__(CS_THREADS) colsum_vec_kernel(const T* __restrict__ X, float* __restrict__ out, int M, int N, int64_t ld,
                                                                 int rows_per_block, int atomic) {
  constexpr int NW = CS_THREADS / 32;
  __shared__ float red[NW][256 + 8];
  __shared__ float part[256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * 256 + lane * 8;
  const int m0 = blockIdx.y * rows_per_block, m1 = min(M, m0 + rows_per_block);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (n < N) {
    int m = m0 + warp;
    for (; m + 3 * NW < m1; m += 4 * NW) {
      float v[4][8];
#pragma unroll
      for (int u = 0; u < 4; u++) ld8(X + (int64_t)(m + u * NW) * ld + n, v[u]);
#pragma unroll
      for (int u = 0; u < 4; u++)
#pragma unroll
        for (int k = 0; k < 8; k++) acc[k] += v[u][k];
    }
    for (; m < m1; m += NW) {
      float v[8];
      ld8(X + (int64_t)m * ld + n, v);
#pragma unroll
      for (int k = 0; k < 8; k++) acc[k] += v[k];
    }
  }
#pragma unroll
  for (int k = 0; k < 8; k++) red[warp][lane * 8 + k] = acc[k];
  __syncthreads();
  const int c = threadIdx.x;
  if (c < 256) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < NW; w++) t += red[w][c];
    part[c] = t;
  }
  cl_sync();
  if (cl_rank() == 0 && c < 256 && blockIdx.x * 256 + c < N) {
    const float t = cl_sum(&part[c]);
    if (atomic) atomicAdd(out + blockIdx.x * 256 + c, t);
    else out[blockIdx.x * 256 + c] += t;
  }
  cl_sync();
}

// any N / ld / alignment: 32 columns per block, 32 row lanes
template <typename T>
__global__ void __launch_bounds__(CS_THREADS) colsum_kernel(const T* __restrict__ X, float* __restrict__ out, int M, int N, int64_t ld,
                                                             int rows_per_block, int atomic) {
  __shared__ float red[32][33];
  const int n = blockIdx.x * 32 + threadIdx.x;
  const int m0 = blockIdx.y * rows_per_block, m1 = min(M, m0 + rows_per_block);
  float s = 0.f;
  if (n < N)
    for (int m = m0 + threadIdx.y; m < m1; m += 32) s += ldf(X + (int64_t)m * ld + n);
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 32; i++) t += red[i][threadIdx.x];
    red[0][threadIdx.x] = t;
  }
  cl_sync();
  if (cl_rank() == 0 && threadIdx.y == 0 && n < N) {
    const float t = cl_sum(&red[0][threadIdx.x]);
    if (atomic) atomicAdd(out + n, t);
    else out[n] += t;
  }
  cl_sync();
}

int colsum(const void* X, int dt, float* out, int M, int N, int64_t ld, int accumulate, cudaStream_t st) {
  LO_CHECK_ARG(M > 0 && N > 0, "empty colsum");
  static bool attr = false;
  if (!attr) {
    LO_CUDA(cudaFuncSetAttribute(colsum_vec_kernel<float>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    LO_CUDA(cudaFuncSetAttribute(colsum_vec_kernel<bf16>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    LO_CUDA(cudaFuncSetAttribute(colsum_kernel<float>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    LO_CUDA(cudaFuncSetAttribute(colsum_kernel<bf16>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    attr = true;
  }
  if (!accumulate) LO_CUDA(cudaMemsetAsync(out, 0, (size_t)N * sizeof(float), st));
  const size_t es = dt == LO_F32 ? 4 : 2;
  const bool vec = N % 8 == 0 && ld % 8 == 0 && ((uintptr_t)X % (8 * es)) == 0;
  const int cb = vec ? cdiv(N, 256) : cdiv(N, 32);
  if (!g_opt_det) {
    int splits = cdiv(LO_NUM_SMS * 2, cb);
    if (splits > cdiv(M, 128)) splits = cdiv(M, 128);
    if (splits < 1) splits = 1;
    const int rpb = cdiv(M, splits);
    const dim3 grid(cb, cdiv(M, rpb));
    if (vec) {
      LO_DISPATCH_DT(dt, T, (colsum_vec_kernel<T><<<grid, CS_THREADS, 0, st>>>((const T*)X, out, M, N, ld, rpb, 1)));
    } else {
      LO_DISPATCH_DT(dt, T, (colsum_kernel<T><<<grid, dim3(32, 32), 0, st>>>((const T*)X, out, M, N, ld, rpb, 1)));
    }
    LO_LAUNCH_OK();
    return LO_OK;
  }
  // ordered: one cluster of up to 16 row splits (>= 256 rows each), a second one only onto the zeroed output
  int cs = cdiv(M, 256);
  if (cs > CS_MAXCL) cs = CS_MAXCL;
  const int groups = (!accumulate && cs == CS_MAXCL && M >= 2 * CS_MAXCL * 256) ? 2 : 1;
  const int rpb = cdiv(M, cs * groups);
  const dim3 grid(cb, cs * groups), cl(1, cs, 1);
  if (vec) {
    LO_DISPATCH_DT(dt, T, LO_CUDA(launch_cluster(colsum_vec_kernel<T>, grid, dim3(CS_THREADS), 0, st, cl, false, (const T*)X, out, M, N, ld,
                                                  rpb, groups > 1 ? 1 : 0)));
  } else {
    LO_DISPATCH_DT(dt, T, LO_CUDA(launch_cluster(colsum_kernel<T>, grid, dim3(32, 32), 0, st, cl, false, (const T*)X, out, M, N, ld, rpb,
                                                  groups > 1 ? 1 : 0)));
  }
  LO_LAUNCH_OK();
  return LO_OK;
}

// the run-time options of lo_common.cuh's LO_OPTIONS and the name table lo_set_option / lo_get_option / lo_option_name walk
#define LO_OPTION_DEFINE(var, name, def) int var = def;
LO_OPTIONS(LO_OPTION_DEFINE)
#undef LO_OPTION_DEFINE

struct Option {
  const char* name;
  int* var;
};
#define LO_OPTION_ENTRY(var, name, def) {name, &var},
static const Option g_options[] = {LO_OPTIONS(LO_OPTION_ENTRY)};
#undef LO_OPTION_ENTRY
constexpr int NUM_OPTIONS = sizeof(g_options) / sizeof(g_options[0]);

static int* find_option(const char* name) {
  for (int i = 0; name && i < NUM_OPTIONS; i++)
    if (!strcmp(name, g_options[i].name)) return g_options[i].var;
  return nullptr;
}

}  // namespace lo

extern "C" {

int lo_version(void) { return 100; }
const char* lo_last_error(void) { return lo::g_err; }
int64_t lo_launch_count(void) { return lo::g_launches; }
int lo_tc_available(void) { return lo::tc_available() ? 1 : 0; }

const char* lo_option_name(int i) { return i >= 0 && i < lo::NUM_OPTIONS ? lo::g_options[i].name : nullptr; }

int lo_get_option(const char* name) {
  const int* v = lo::find_option(name);
  return v ? *v : -1;
}

int lo_set_option(const char* name, int value) {
  int* v = lo::find_option(name);
  if (!v) return lo::fail(LO_EINVAL, "lo_set_option: unknown option %s", name ? name : "(null)");
  if (v == &lo::g_opt_l2_persist_mb) {
    // an action: size of the L2 set-aside that evict_last / persisting accesses may occupy (0 = driver default)
    cudaError_t e = cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, (size_t)value << 20);
    if (e != cudaSuccess) return lo::fail(LO_ECUDA, "lo_set_option(l2_persist_mb): %s (%ld)", cudaGetErrorString(e), (long)e);
  }
  *v = value;
  return LO_OK;
}

int lo_gemm(const void* A, int dtA, const void* B, int dtB, void* C, int dtC, int M, int N, int K, int64_t sam,
            int64_t sak, int64_t sbk, int64_t sbn, int64_t ldc, int batch, int64_t sA, int64_t sB, int64_t sC,
            const float* bias, int accumulate, int relu, int impl, void* stream) {
  LO_CHECK_ARG(A && B && C, "null pointer");
  lo::GemmDesc d{M, N, K, sam, sak, sbk, sbn, ldc, batch, sA, sB, sC, bias, accumulate, relu};
  return lo::gemm(A, dtA, B, dtB, C, dtC, d, impl, (cudaStream_t)stream);
}

int lo_colsum(const void* X, int dt, float* out, int M, int N, int64_t ld, int accumulate, void* stream) {
  LO_CHECK_ARG(X && out, "null pointer");
  return lo::colsum(X, dt, out, M, N, ld, accumulate, (cudaStream_t)stream);
}

}  // extern "C"
