// Self-critical sequence training (Rennie et al. 2017) of both decoder flavours: the edit-distance reward of a sample and of
// the greedy rollout, and the policy gradient of the sample's log-probability (include/latex_ocr_b200.h, lo_scst_*; the _tf entry
// points take the TF layout).  The sample itself is drawn inside the decoder's time loop (ss_block_tokens, lo_decoder.cu).
#include "lo_common.cuh"

namespace lo {

constexpr int SCST_MAX_LEN = 512;

// length of s[0..L) truncated at its first end_id (metrics.truncate_end); one warp
__device__ __forceinline__ int trunc_len(const int64_t* s, int L, int64_t end_id) {
  const int lane = threadIdx.x & 31;
  for (int base = 0; base < L; base += 32) {
    const int i = base + lane;
    const unsigned m = __ballot_sync(0xffffffffu, i < L && s[i] == end_id);
    if (m) return base + __ffs(m) - 1;
  }
  return L;
}

// unit-cost Levenshtein distance of h[0..n) and r[0..m) (shared memory), one warp.  It sweeps the anti-diagonals k = i + j of the
// (n+1) x (m+1) table: cell (i, j) needs (i-1, j-1) from diagonal k-2 and (i-1, j), (i, j-1) from diagonal k-1.  d0 / d1 / d2 hold
// diagonals k-2 / k-1 / k indexed by i (n + 1 ints each).  Integer arithmetic: exact.
__device__ int warp_levenshtein(const int64_t* h, int n, const int64_t* r, int m, int* d0, int* d1, int* d2) {
  const int lane = threadIdx.x & 31;
  for (int k = 0; k <= n + m; k++) {
    const int lo = max(0, k - m), hi = min(n, k);
    for (int i = lo + lane; i <= hi; i += 32) {
      const int j = k - i;
      d2[i] = i == 0 ? j : (j == 0 ? i : min(d0[i - 1] + (h[i - 1] != r[j - 1] ? 1 : 0), min(d1[i - 1], d1[i]) + 1));
    }
    __syncwarp();
    int* t = d0;
    d0 = d1;
    d1 = d2;
    d2 = t;
  }
  return d1[n];
}

// One block per row: warp 0 scores the sample, warp 1 the greedy rollout.  Dynamic shared memory: ref [Lr] | hyp [Lh] | greedy [Lg]
// int64, then three diagonals of Lmax = max(Lh, Lg) + 1 ints per warp.  s0: the first position of hyp that was drawn (1 in the
// torch layout, where hyp[0] is the given start token; 0 in the TF layout).
__global__ void __launch_bounds__(64) scst_reward_kernel(const int64_t* __restrict__ hyp, int64_t hs, int Lh,
                                                         const int64_t* __restrict__ greedy, int64_t gs, int Lg,
                                                         const int64_t* __restrict__ ref, int64_t rs, int Lr, int64_t end_id,
                                                         int s0, float* __restrict__ r_sample, float* __restrict__ r_greedy,
                                                         float* __restrict__ adv, int32_t* __restrict__ n_len) {
  extern __shared__ int64_t sm[];
  __shared__ float s_r[2];
  const int b = blockIdx.x, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Lmax = max(Lh, Lg) + 1;
  int64_t* s_ref = sm;
  int64_t* s_h = s_ref + Lr;
  int64_t* s_g = s_h + Lh;
  int* diag = (int*)(s_g + Lg) + w * 3 * Lmax;
  for (int i = threadIdx.x; i < Lr; i += blockDim.x) s_ref[i] = ref[(int64_t)b * rs + i];
  for (int i = threadIdx.x; i < Lh; i += blockDim.x) s_h[i] = hyp[(int64_t)b * hs + i];
  if (greedy)
    for (int i = threadIdx.x; i < Lg; i += blockDim.x) s_g[i] = greedy[(int64_t)b * gs + i];
  __syncthreads();
  if (w == 0 || greedy) {
    const int64_t* h = w == 0 ? s_h : s_g;
    const int n = trunc_len(h, w == 0 ? Lh : Lg, end_id), m = trunc_len(s_ref, Lr, end_id);
    const int dist = warp_levenshtein(h, n, s_ref, m, diag, diag + Lmax, diag + 2 * Lmax);
    const int mx = max(n, m);
    // metrics.edit_distance's per-row value, rounded once from double
    if (lane == 0) s_r[w] = mx == 0 ? 1.f : (float)(1.0 - (double)dist / (double)mx);
  }
  // n_b = the number of draws up to and including the first END: torch (s0 = 1) the first t >= 1 with hyp[t] == end_id, else
  // Lh - 1; TF (s0 = 0) that t + 1 for t >= 0, else Lh
  const int nb = w == 0 ? min(1 + trunc_len(s_h + s0, Lh - s0, end_id), Lh - s0) : 0;
  __syncthreads();
  if (threadIdx.x == 0) {
    r_sample[b] = s_r[0];
    if (greedy && r_greedy) r_greedy[b] = s_r[1];
    if (greedy && adv) adv[b] = s_r[0] - s_r[1];
    if (n_len) n_len[b] = nb;
  }
}

// block-wide reduction of a 128-thread block in a fixed order (MAX: maximum, else sum)
template <bool MAX>
__device__ __forceinline__ float block_reduce128(float x, float* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float y = __shfl_xor_sync(0xffffffffu, x, o);
    x = MAX ? fmaxf(x, y) : x + y;
  }
  __syncthreads();                 // sh may still be read by the previous reduction
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = x;
  __syncthreads();
  return MAX ? fmaxf(fmaxf(sh[0], sh[1]), fmaxf(sh[2], sh[3])) : (sh[0] + sh[1]) + (sh[2] + sh[3]);
}

// One block per prediction row (s, b): the softmax of preds / tau, d L / d preds into dpred (batch-major rows ds apart), and the
// row's log pi(fed[b][s + foff]) into partial (0 past the row's n_b).  Row (s, b) of preds is at b * pb + s * pt: torch
// (batch-major, s = t - 1, foff = 1) or TF (time-major, s = t, foff = 0).
__global__ void __launch_bounds__(128) scst_pg_kernel(const float* __restrict__ preds, int64_t pb, int64_t pt,
                                                      const int64_t* __restrict__ fed, int64_t fs, int foff, const float* __restrict__ adv,
                                                      const int32_t* __restrict__ n_len, const float* __restrict__ temp, int T, int V,
                                                      float inv_B, float* __restrict__ dpred, int64_t ds, float* __restrict__ partial) {
  __shared__ float sh[4];
  const int s = blockIdx.x, b = blockIdx.y;
  float* out = dpred + ((int64_t)b * T + s) * ds;
  if (s >= n_len[b]) {             // no draw of this row enters L (the last row never does)
    for (int v = threadIdx.x; v < V; v += blockDim.x) out[v] = 0.f;
    if (threadIdx.x == 0) partial[(int64_t)b * T + s] = 0.f;
    return;
  }
  const float* x = preds + (int64_t)b * pb + (int64_t)s * pt;
  const float tau = *temp;
  float mx = -INFINITY;
  for (int v = threadIdx.x; v < V; v += blockDim.x) mx = fmaxf(mx, x[v] / tau);
  mx = block_reduce128<true>(mx, sh);
  float sum = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) sum += expf(x[v] / tau - mx);
  const float lse = mx + logf(block_reduce128<false>(sum, sh));
  int64_t f = fed[(int64_t)b * fs + s + foff];
  f = f < 0 ? 0 : (f >= V ? V - 1 : f);        // the token the cell embedded (lstm_pw_fwd_body clamps it the same way)
  const float g = -adv[b] * inv_B / tau;
  for (int v = threadIdx.x; v < V; v += blockDim.x) out[v] = g * ((v == f ? 1.f : 0.f) - expf(x[v] / tau - lse));
  if (threadIdx.x == 0) partial[(int64_t)b * T + s] = x[f] / tau - lse;
}

// stats = {L, mean r_sample, mean r_greedy, mean n_len}: each thread sums its rows' partials in step order, then a fixed tree
__global__ void __launch_bounds__(256) scst_loss_kernel(const float* __restrict__ partial, const float* __restrict__ adv,
                                                        const int32_t* __restrict__ n_len, const float* __restrict__ r_s,
                                                        const float* __restrict__ r_g, int B, int T, float* __restrict__ stats) {
  __shared__ float sh[4][256];
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    float lp = 0.f;
    for (int s = 0; s < T; s++) lp += partial[(int64_t)b * T + s];
    acc[0] += adv[b] * lp;
    acc[1] += r_s ? r_s[b] : 0.f;
    acc[2] += r_g ? r_g[b] : 0.f;
    acc[3] += (float)n_len[b];
  }
#pragma unroll
  for (int q = 0; q < 4; q++) sh[q][threadIdx.x] = acc[q];
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h)
#pragma unroll
      for (int q = 0; q < 4; q++) sh[q][threadIdx.x] += sh[q][threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    stats[0] = -sh[0][0] / (float)B;
    stats[1] = sh[1][0] / (float)B;
    stats[2] = sh[2][0] / (float)B;
    stats[3] = sh[3][0] / (float)B;
  }
}

}  // namespace lo

using namespace lo;

// the entry points: torch layout (s0 = 1, foff = 1, batch-major preds) and TF layout (s0 = 0, foff = 0, time-major logits)
static int edit_reward(const int64_t* hyp, int64_t hyp_stride, int Lh, const int64_t* greedy, int64_t greedy_stride, int Lg,
                       const int64_t* ref, int64_t ref_stride, int Lr, int B, int64_t end_id, int s0, float* r_sample, float* r_greedy,
                       float* adv, int32_t* n_len, void* stream) {
  LO_CHECK_ARG(hyp && ref && r_sample, "null pointer");
  LO_CHECK_ARG(B >= 1, "B >= 1");
  LO_CHECK_ARG(Lh >= 1 && Lh <= SCST_MAX_LEN && Lr >= 1 && Lr <= SCST_MAX_LEN, "hypothesis / reference lengths in 1..512");
  LO_CHECK_ARG(!greedy || (Lg >= 1 && Lg <= SCST_MAX_LEN), "greedy length in 1..512");
  LO_CHECK_ARG(hyp_stride >= Lh && ref_stride >= Lr && (!greedy || greedy_stride >= Lg), "row strides >= lengths");
  if (!greedy) Lg = 0;
  const size_t smem = (size_t)(Lr + Lh + Lg) * 8 + (size_t)2 * 3 * (max(Lh, Lg) + 1) * 4;
  scst_reward_kernel<<<B, 64, smem, (cudaStream_t)stream>>>(hyp, hyp_stride, Lh, greedy, greedy_stride, Lg, ref, ref_stride, Lr, end_id,
                                                            s0, r_sample, r_greedy, adv, n_len);
  LO_LAUNCH_OK();
  return LO_OK;
}

static int pg_grad(const float* preds, int64_t pb, int64_t pt, int64_t pred_stride, const int64_t* fed, int64_t fed_stride, int foff,
                   const float* adv, const int32_t* n_len, const float* temp, const float* r_sample, const float* r_greedy, int B, int T,
                   int V, float* dpred, int64_t dpred_stride, float* partial, float* stats, void* stream) {
  LO_CHECK_ARG(preds && fed && adv && n_len && temp && dpred && partial && stats, "null pointer");
  LO_CHECK_ARG(B >= 1 && T >= 1 && V >= 2 && T <= 65535, "B, T >= 1, T <= 65535, V >= 2");
  LO_CHECK_ARG(pred_stride >= V && dpred_stride >= V && fed_stride >= T, "pred_stride, dpred_stride >= V; fed_stride >= T");
  cudaStream_t st = (cudaStream_t)stream;
  scst_pg_kernel<<<dim3(T, B), 128, 0, st>>>(preds, pb, pt, fed, fed_stride, foff, adv, n_len, temp, T, V, 1.0f / (float)B, dpred,
                                             dpred_stride, partial);
  LO_LAUNCH_OK();
  scst_loss_kernel<<<1, 256, 0, st>>>(partial, adv, n_len, r_sample, r_greedy, B, T, stats);
  LO_LAUNCH_OK();
  return LO_OK;
}

extern "C" int lo_scst_edit_reward(const int64_t* hyp, int64_t hyp_stride, int Lh, const int64_t* greedy, int64_t greedy_stride,
                                   int Lg, const int64_t* ref, int64_t ref_stride, int Lr, int B, int64_t end_id, float* r_sample,
                                   float* r_greedy, float* adv, int32_t* n_len, void* stream) {
  return edit_reward(hyp, hyp_stride, Lh, greedy, greedy_stride, Lg, ref, ref_stride, Lr, B, end_id, 1, r_sample, r_greedy, adv, n_len,
                     stream);
}

extern "C" int lo_scst_edit_reward_tf(const int64_t* hyp, int64_t hyp_stride, int Lh, const int64_t* greedy, int64_t greedy_stride,
                                      int Lg, const int64_t* ref, int64_t ref_stride, int Lr, int B, int64_t end_id, float* r_sample,
                                      float* r_greedy, float* adv, int32_t* n_len, void* stream) {
  return edit_reward(hyp, hyp_stride, Lh, greedy, greedy_stride, Lg, ref, ref_stride, Lr, B, end_id, 0, r_sample, r_greedy, adv, n_len,
                     stream);
}

extern "C" int lo_scst_pg_grad(const float* preds, int64_t pred_stride, const int64_t* fed, int64_t fed_stride, const float* adv,
                               const int32_t* n_len, const float* temp, const float* r_sample, const float* r_greedy, int B, int T,
                               int V, float* dpred, int64_t dpred_stride, float* partial, float* stats, void* stream) {
  return pg_grad(preds, (int64_t)T * pred_stride, pred_stride, pred_stride, fed, fed_stride, 1, adv, n_len, temp, r_sample, r_greedy, B,
                 T, V, dpred, dpred_stride, partial, stats, stream);
}

extern "C" int lo_scst_pg_grad_tf(const float* logits, int64_t ldl, const int64_t* fed, int64_t fed_stride, const float* adv,
                                  const int32_t* n_len, const float* temp, const float* r_sample, const float* r_greedy, int B, int T,
                                  int V, float* dpred, int64_t dpred_stride, float* partial, float* stats, void* stream) {
  return pg_grad(logits, ldl, (int64_t)B * ldl, ldl, fed, fed_stride, 0, adv, n_len, temp, r_sample, r_greedy, B, T, V, dpred,
                 dpred_stride, partial, stats, stream);
}
