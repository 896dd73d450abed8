// Attention-LSTM decoder of the torch flavour (DecoderWithAttention, seq2seq_torch.py:195-320) with the
// loss of img2seq_torch.py:147-159: forward over T teacher-forced steps, hand-derived backward.
//
// Schedule (see DESIGN.md §4): everything that does not depend on the recurrence is hoisted out of the
// time loop (att1 = encoder_att(enc), the embedding->gate projection table, logits, every weight
// gradient, d att1 and d enc).  Inside the loop each step reads enc and att1 exactly ONCE in forward
// and ONCE in backward (the HBM roofline of SURVEY.md §8-d) and runs two skinny GEMMs.
#include "lo_common.cuh"
#include "lo_ptx.cuh"

namespace lo {

#define LO_ATT_THREADS 256
#define LO_ATT_WARPS 8
#define LO_ATT_MAXSPLIT 16

static inline int att_splits(int B) {
  int s = (444 + B - 1) / B;
  if (s < 1) s = 1;
  if (s > LO_ATT_MAXSPLIT) s = LO_ATT_MAXSPLIT;
  return s;
}

__device__ __forceinline__ float ldcg_f(const float* p) { return __ldcg(p); }

// ------------------------------------------------------------------------------------------------
// K5: attention forward for one step.  grid (nsplit, B), 256 threads.  Each warp streams rows of
// att1 and enc (16 B per lane per load), keeps an online-softmax state (m, l, acc[C/32]) in registers;
// CTA combine in smem, cross-CTA combine by the last CTA to finish (threadfence + ticket).
// NV = A/256 = C/256 vectors of 8 elements per lane.
// ------------------------------------------------------------------------------------------------
template <typename T, int NV>
__global__ void __launch_bounds__(LO_ATT_THREADS) attention_fwd_kernel(
    const T* __restrict__ att1, const T* __restrict__ enc, const float* __restrict__ att2, int64_t att2_stride,
    const float* __restrict__ wf, float* __restrict__ alpha, int64_t alpha_stride, float* __restrict__ ctx,
    float* __restrict__ gate_pre, int64_t gate_stride, float* __restrict__ gctx, bf16* __restrict__ gctx_bf, int R, int nsplit,
    int* __restrict__ counters, float* __restrict__ partials, int rpi) {
  constexpr int CH = NV * 256;   // A == C == CH
  const int b = blockIdx.y, sp = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int rps = (R + nsplit - 1) / nsplit;
  const int r0 = sp * rps, r1 = min(R, r0 + rps);
  float a2[NV * 8], wv[NV * 8], acc[NV * 8];
#pragma unroll
  for (int j = 0; j < NV; j++) {
    ld8(att2 + (int64_t)b * att2_stride + (j * 32 + lane) * 8, a2 + j * 8);
    ld8(wf + (j * 32 + lane) * 8, wv + j * 8);
#pragma unroll
    for (int i = 0; i < 8; i++) acc[j * 8 + i] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  const T* a1b = att1 + (int64_t)(b / rpi) * R * CH;
  const T* eb = enc + (int64_t)(b / rpi) * R * CH;
  float* alb = alpha + (int64_t)b * alpha_stride;
  for (int r = r0 + wid; r < r1; r += 2 * LO_ATT_WARPS) {
    const int rb = r + LO_ATT_WARPS;
    const bool two = rb < r1;
    float v0[NV * 8], v1[NV * 8], u0[NV * 8], u1[NV * 8];
#pragma unroll
    for (int j = 0; j < NV; j++) {
      ld8(a1b + (int64_t)r * CH + (j * 32 + lane) * 8, v0 + j * 8);
      ld8(eb + (int64_t)r * CH + (j * 32 + lane) * 8, u0 + j * 8);
    }
    if (two) {
#pragma unroll
      for (int j = 0; j < NV; j++) {
        ld8(a1b + (int64_t)rb * CH + (j * 32 + lane) * 8, v1 + j * 8);
        ld8(eb + (int64_t)rb * CH + (j * 32 + lane) * 8, u1 + j * 8);
      }
    }
    float e0 = 0.f, e1 = 0.f;
#pragma unroll
    for (int i = 0; i < NV * 8; i++) {
      e0 = fmaf(wv[i], fmaxf(v0[i] + a2[i], 0.f), e0);
      if (two) e1 = fmaf(wv[i], fmaxf(v1[i] + a2[i], 0.f), e1);
    }
    e0 = warp_sum(e0);
    e1 = warp_sum(e1);
    if (lane == 0) {
      alb[r] = e0;
      if (two) alb[rb] = e1;
    }
    const float mn = two ? fmaxf(m, fmaxf(e0, e1)) : fmaxf(m, e0);
    const float sc = expf(m - mn);     // m = -inf on the first row -> 0
    const float p0 = expf(e0 - mn);
    const float p1 = two ? expf(e1 - mn) : 0.f;
    l = l * sc + p0 + p1;
#pragma unroll
    for (int i = 0; i < NV * 8; i++) {
      float t = acc[i] * sc;
      t = fmaf(p0, u0[i], t);
      if (two) t = fmaf(p1, u1[i], t);
      acc[i] = t;
    }
    m = mn;
  }
  // ---- CTA combine
  __shared__ float s_m[LO_ATT_WARPS], s_l[LO_ATT_WARPS];
  __shared__ float s_acc[LO_ATT_WARPS][CH];
  __shared__ float s_scale[LO_ATT_MAXSPLIT];
  __shared__ float s_ML[2];
  __shared__ int s_last;
  if (lane == 0) { s_m[wid] = m; s_l[wid] = l; }
#pragma unroll
  for (int j = 0; j < NV; j++)
#pragma unroll
    for (int i = 0; i < 8; i++) s_acc[wid][(j * 32 + lane) * 8 + i] = acc[j * 8 + i];
  __syncthreads();
  float M = -INFINITY;
#pragma unroll
  for (int w = 0; w < LO_ATT_WARPS; w++) M = fmaxf(M, s_m[w]);
  float L = 0.f;
  float wsc[LO_ATT_WARPS];
#pragma unroll
  for (int w = 0; w < LO_ATT_WARPS; w++) {
    wsc[w] = (s_m[w] == -INFINITY) ? 0.f : expf(s_m[w] - M);
    L += s_l[w] * wsc[w];
  }
  float* part = partials + ((int64_t)b * nsplit + sp) * (CH + 2);
  for (int c = threadIdx.x; c < CH; c += LO_ATT_THREADS) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < LO_ATT_WARPS; w++) t = fmaf(s_acc[w][c], wsc[w], t);
    part[2 + c] = t;
  }
  if (threadIdx.x == 0) { part[0] = M; part[1] = L; }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int ticket = atomicAdd(counters + b, 1);
    s_last = (ticket == nsplit - 1);
    if (s_last) counters[b] = 0;   // ready for the next launch
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- last CTA of this batch row: global combine, write ctx (+gate), normalise alpha
  const float* pb = partials + (int64_t)b * nsplit * (CH + 2);
  if (threadIdx.x == 0) {
    float Mg = -INFINITY;
    for (int s = 0; s < nsplit; s++) Mg = fmaxf(Mg, ldcg_f(pb + (int64_t)s * (CH + 2)));
    float Lg = 0.f;
    for (int s = 0; s < nsplit; s++) {
      const float ms = ldcg_f(pb + (int64_t)s * (CH + 2));
      const float scl = (ms == -INFINITY) ? 0.f : expf(ms - Mg);
      s_scale[s] = scl;
      Lg += ldcg_f(pb + (int64_t)s * (CH + 2) + 1) * scl;
    }
    s_ML[0] = Mg;
    s_ML[1] = 1.0f / Lg;
  }
  __syncthreads();
  const float Mg = s_ML[0], invL = s_ML[1];
  for (int c = threadIdx.x; c < CH; c += LO_ATT_THREADS) {
    float t = 0.f;
    for (int s = 0; s < nsplit; s++) t = fmaf(ldcg_f(pb + (int64_t)s * (CH + 2) + 2 + c), s_scale[s], t);
    t *= invL;
    ctx[(int64_t)b * CH + c] = t;
    if (gate_pre) {
      const float g = sigmoidf_(gate_pre[(int64_t)b * gate_stride + c]);
      gate_pre[(int64_t)b * gate_stride + c] = g;
      gctx[(int64_t)b * CH + c] = g * t;
      if (gctx_bf) gctx_bf[(int64_t)b * CH + c] = __float2bfloat16_rn(g * t);
    }
  }
  for (int r = threadIdx.x; r < R; r += LO_ATT_THREADS) alb[r] = expf(ldcg_f(alb + r) - Mg) * invL;
}

// ------------------------------------------------------------------------------------------------
// K6: attention backward for one step (same streaming structure; reads enc and att1 once).
//   dctx = dgctx*gate ; dgp = dgctx*ctx*gate*(1-gate) ; s = <dctx,ctx> + sreg
//   dalpha_r = <dctx, enc_r> + dreg_r ; de_r = alpha_r (dalpha_r - s) ; datt2_a = wf_a sum_r de_r [att1_ra + att2_a > 0]
// ------------------------------------------------------------------------------------------------
template <typename T, int NV>
__global__ void __launch_bounds__(LO_ATT_THREADS) attention_bwd_kernel(
    const T* __restrict__ att1, const T* __restrict__ enc, const float* __restrict__ att2, const float* __restrict__ gate,
    int64_t o1_stride, const float* __restrict__ wf, const float* __restrict__ alpha, int64_t alpha_stride,
    const float* __restrict__ ctx, const float* __restrict__ dgctx, int64_t dg_stride, const float* __restrict__ dreg,
    int64_t dreg_stride, const float* __restrict__ sreg, int64_t sreg_stride, float* __restrict__ de, float* __restrict__ datt2,
    float* __restrict__ dgp, int64_t dcat_stride, bf16* __restrict__ datt2_bf, bf16* __restrict__ dgp_bf,
    float* __restrict__ dctx_out, int R, int nsplit, int* __restrict__ counters, float* __restrict__ partials) {
  constexpr int CH = NV * 256;
  const int b = blockIdx.y, sp = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int rps = (R + nsplit - 1) / nsplit;
  const int r0 = sp * rps, r1 = min(R, r0 + rps);
  float a2[NV * 8], dc[NV * 8], macc[NV * 8];
  float sdot = 0.f;
#pragma unroll
  for (int j = 0; j < NV; j++) {
    const int c0 = (j * 32 + lane) * 8;
    float g[8], cx[8], dg[8];
    ld8(att2 + (int64_t)b * o1_stride + c0, a2 + j * 8);
    ld8(gate + (int64_t)b * o1_stride + c0, g);
    ld8(ctx + (int64_t)b * CH + c0, cx);
    ld8(dgctx + (int64_t)b * dg_stride + c0, dg);
    float gp[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
      dc[j * 8 + i] = dg[i] * g[i];
      sdot = fmaf(dc[j * 8 + i], cx[i], sdot);
      gp[i] = dg[i] * cx[i] * g[i] * (1.f - g[i]);
      macc[j * 8 + i] = 0.f;
    }
    if (sp == 0 && wid == 0) {
      st8(dgp + (int64_t)b * dcat_stride + c0, gp);
      if (dgp_bf) st8(dgp_bf + (int64_t)b * dcat_stride + c0, gp);
      st8(dctx_out + (int64_t)b * CH + c0, dc + j * 8);
    }
  }
  const float s = warp_sum(sdot) + sreg[(int64_t)b * sreg_stride];
  const T* a1b = att1 + (int64_t)b * R * CH;
  const T* eb = enc + (int64_t)b * R * CH;
  const float* alb = alpha + (int64_t)b * alpha_stride;
  float* deb = de + (int64_t)b * alpha_stride;
  const float* drb = dreg + (int64_t)b * dreg_stride;
  for (int r = r0 + wid; r < r1; r += 2 * LO_ATT_WARPS) {
    const int rb = r + LO_ATT_WARPS;
    const bool two = rb < r1;
    float v0[NV * 8], v1[NV * 8], u0[NV * 8], u1[NV * 8];
#pragma unroll
    for (int j = 0; j < NV; j++) {
      ld8(eb + (int64_t)r * CH + (j * 32 + lane) * 8, u0 + j * 8);
      ld8(a1b + (int64_t)r * CH + (j * 32 + lane) * 8, v0 + j * 8);
    }
    if (two) {
#pragma unroll
      for (int j = 0; j < NV; j++) {
        ld8(eb + (int64_t)rb * CH + (j * 32 + lane) * 8, u1 + j * 8);
        ld8(a1b + (int64_t)rb * CH + (j * 32 + lane) * 8, v1 + j * 8);
      }
    }
    float d0 = 0.f, d1 = 0.f;
#pragma unroll
    for (int i = 0; i < NV * 8; i++) {
      d0 = fmaf(dc[i], u0[i], d0);
      if (two) d1 = fmaf(dc[i], u1[i], d1);
    }
    d0 = warp_sum(d0);
    d1 = warp_sum(d1);
    const float de0 = alb[r] * (d0 + drb[r] - s);
    const float de1 = two ? alb[rb] * (d1 + drb[rb] - s) : 0.f;
    if (lane == 0) {
      deb[r] = de0;
      if (two) deb[rb] = de1;
    }
#pragma unroll
    for (int i = 0; i < NV * 8; i++) {
      macc[i] += (v0[i] + a2[i] > 0.f) ? de0 : 0.f;
      if (two) macc[i] += (v1[i] + a2[i] > 0.f) ? de1 : 0.f;
    }
  }
  __shared__ float s_acc[LO_ATT_WARPS][CH];
  __shared__ int s_last;
#pragma unroll
  for (int j = 0; j < NV; j++)
#pragma unroll
    for (int i = 0; i < 8; i++) s_acc[wid][(j * 32 + lane) * 8 + i] = macc[j * 8 + i];
  __syncthreads();
  float* part = partials + ((int64_t)b * nsplit + sp) * (CH + 2);
  for (int c = threadIdx.x; c < CH; c += LO_ATT_THREADS) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < LO_ATT_WARPS; w++) t += s_acc[w][c];
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
  const float* pb = partials + (int64_t)b * nsplit * (CH + 2);
  for (int c = threadIdx.x; c < CH; c += LO_ATT_THREADS) {
    float t = 0.f;
    for (int sidx = 0; sidx < nsplit; sidx++) t += ldcg_f(pb + (int64_t)sidx * (CH + 2) + 2 + c);
    datt2[(int64_t)b * dcat_stride + c] = t * wf[c];
    if (datt2_bf) datt2_bf[(int64_t)b * dcat_stride + c] = __float2bfloat16_rn(t * wf[c]);
  }
}

// ------------------------------------------------------------------------------------------------
// hoisted d att1 / d w_full: ONE sweep over att1 after the time loop.
//   datt1[b,r,a] = wf[a] * sum_t de[b,t,r] * [att1[b,r,a] + att2[t,b,a] > 0]
//   dwf[a]      += sum_{b,r,t} de[b,t,r] * relu(att1[b,r,a] + att2[t,b,a])
// grid (A/64, ceil(R/(32 nchunk)), B), 128 threads, thread tile 4(r) x 4(a), time chunks of 32 staged in smem.  d w_full: each
// block adds its sums onto dwf[A] with fp32 atomics, or (dwf_rows, option "deterministic") the row blocks of a batch row (<= 16)
// form one cluster and dwf is a [B][A] scratch (row b += that batch row's sum, added in block order).
// ------------------------------------------------------------------------------------------------
// WACC: 0 = d att1 only; 1 = also all of d w_full; 2 = only the `x * (sum_t on * de)` term of d w_full (ReLU): the other term,
// sum_{t,b} att2_t[b,a] * sum_r on * de_t[b,r], was accumulated per step by the mask-bit attention backward kernels (dwf_part)
template <typename T, int WACC, int ACT = 0>
__global__ void __launch_bounds__(128) datt1_kernel(const T* __restrict__ att1, const float* __restrict__ out1,
                                                     int64_t o1_row, int64_t o1_step, const float* __restrict__ de,
                                                     const float* __restrict__ wf, T* __restrict__ datt1,
                                                     float* __restrict__ dwf, int Tn, int R, int A, int nchunk, int dwf_rows) {
  constexpr int TT = 32;
  __shared__ __align__(16) float s_a2[TT][64];
  __shared__ __align__(16) float s_de[TT][32];
  __shared__ float s_w[8][64];
  const int b = blockIdx.z, a0 = blockIdx.x * 64;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;   // a = a0 + tx*4.., r = r0 + ty*4..
  float wacc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int ch = 0; ch < nchunk; ch++) {                     // 32-row chunks of this block, in order
  const int r0 = (blockIdx.y * nchunk + ch) * 32;
  if (r0 >= R) break;
  float x[4][4], nx[4][4], acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int r = r0 + ty * 4 + i;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      acc[i][j] = 0.f;
      x[i][j] = (r < R) ? ldf(att1 + ((int64_t)b * R + r) * A + a0 + tx * 4 + j) : -INFINITY;
      nx[i][j] = -x[i][j];
    }
  }
  for (int t0 = 0; t0 < Tn; t0 += TT) {
    for (int i = threadIdx.x; i < TT * 64; i += 128) {
      const int tt = i / 64, a = i % 64;
      s_a2[tt][a] = (t0 + tt < Tn) ? out1[(int64_t)(t0 + tt) * o1_step + (int64_t)b * o1_row + a0 + a] : 0.f;
    }
    for (int i = threadIdx.x; i < TT * 32; i += 128) {
      const int tt = i / 32, r = i % 32;
      s_de[tt][r] = (t0 + tt < Tn && r0 + r < R) ? de[((int64_t)b * Tn + t0 + tt) * R + r0 + r] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int tt = 0; tt < TT; tt++) {
      const float4 q = *reinterpret_cast<const float4*>(&s_a2[tt][tx * 4]);
      const float4 d4 = *reinterpret_cast<const float4*>(&s_de[tt][ty * 4]);
      const float a2v[4] = {q.x, q.y, q.z, q.w}, dv[4] = {d4.x, d4.y, d4.z, d4.w};
      if constexpr (ACT == 0 && WACC == 1) {
        // d w_full[a] = sum de * relu(x + a2) = sum_i x[i][a] * (sum_t on * de) + sum_t a2_t[a] * (sum_i on * de): the first term is
        // x * acc at the very end (x does not depend on t), the second needs only the per-step column sums s[j]
        float sc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) {
            const bool on = a2v[j] > nx[i][j];
            if (on) { acc[i][j] += dv[i]; sc[j] += dv[i]; }
          }
#pragma unroll
        for (int j = 0; j < 4; j++) wacc[j] = fmaf(a2v[j], sc[j], wacc[j]);
      } else
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
          if constexpr (ACT == 0) {
            // x + a2 > 0  <=>  a2 > -x exactly (an fp32 sum has the sign of the exact sum): one compare + one predicated add
            const bool on = a2v[j] > nx[i][j];
            acc[i][j] += on ? dv[i] : 0.f;
          } else {
            const float pre = x[i][j] + a2v[j];
            // tanh score (Genthial cell); padded rows: tanh(-inf) = -1 -> derivative 0, dv = 0
            const float post = tanhf(pre);
            acc[i][j] = fmaf(dv[i], 1.f - post * post, acc[i][j]);
            if (WACC) wacc[j] = fmaf(dv[i], post, wacc[j]);
          }
        }
    }
    __syncthreads();
  }
  float wv[4];
#pragma unroll
  for (int j = 0; j < 4; j++) wv[j] = wf[a0 + tx * 4 + j];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int r = r0 + ty * 4 + i;
    if (r >= R) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) stf(datt1 + ((int64_t)b * R + r) * A + a0 + tx * 4 + j, acc[i][j] * wv[j]);
  }
  if constexpr (WACC != 0 && ACT == 0) {
#pragma unroll
    for (int i = 0; i < 4; i++)
      if (r0 + ty * 4 + i < R) {
#pragma unroll
        for (int j = 0; j < 4; j++) wacc[j] = fmaf(x[i][j], acc[i][j], wacc[j]);      // the x * (sum_t on * de) term
      }
  }
  }
  if (!WACC) return;
#pragma unroll
  for (int j = 0; j < 4; j++) s_w[ty][tx * 4 + j] = wacc[j];
  __syncthreads();
  if (threadIdx.x < 64) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; k++) t += s_w[k][threadIdx.x];
    s_w[0][threadIdx.x] = t;
  }
  if (!dwf_rows) {
    if (threadIdx.x < 64) atomicAdd(dwf + a0 + threadIdx.x, s_w[0][threadIdx.x]);
    return;
  }
  // ordered: the row blocks of batch row b are one cluster; rank 0 adds their sums in order onto the row's [B][A] scratch (one
  // writer per element; the caller sums the rows over b with colsum)
  cl_sync();
  if (cl_rank() == 0 && threadIdx.x < 64) dwf[(int64_t)b * A + a0 + threadIdx.x] += cl_sum(&s_w[0][threadIdx.x]);
  cl_sync();
}

// ------------------------------------------------------------------------------------------------
// small pointwise / reduction kernels
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void mean_rows_kernel(const T* __restrict__ enc, float* __restrict__ mean, int R, int C, int rpi) {
  const int b = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int r = 0; r < R; r++) s += ldf(enc + ((int64_t)(b / rpi) * R + r) * C + c);
  mean[(int64_t)b * C + c] = s / (float)R;
}
// the same over the packed layout (lo_decoder_args.reg_off): row b averages its image's own regions, in mean_rows_kernel's order
template <typename T>
__global__ void mean_segments_kernel(const T* __restrict__ enc, float* __restrict__ mean, const int32_t* __restrict__ reg_off, int C,
                                     int rpi) {
  const int b = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int g0 = reg_off[b / rpi], R = reg_off[b / rpi + 1] - g0;
  float s = 0.f;
  for (int r = 0; r < R; r++) s += ldf(enc + ((int64_t)g0 + r) * C + c);
  mean[(int64_t)b * C + c] = s / (float)R;
}

// scheduled-sampling operands of lstm_pw_fwd_kernel<true> (row pointers at the first row of the launch, step t)
struct SsStep {
  const float* prev_logits;   // logits of step t-1 (NULL at t = 0), rows lstride apart
  int64_t lstride;
  const float* prob;          // device scalar p
  const float* u;             // injected uniforms of step t, rows ustride apart, or NULL: Philox keyed by coin_state
  const unsigned long long* coin_state;   // {seed, call} (lo_decoder_args.dropout_state)
  int64_t ustride;
  int64_t* fed;               // fed tokens of step t, rows ustride apart
  bf16* hd_bf;                // bf16 mirror of hd (A operand of the per-step fc GEMM in bf16), NULL otherwise
};

// the categorical draw of lstm_pw_fwd_gumbel_kernel (lo_decoder_args.ss_temp)
struct GumbelStep {
  const float* temp;          // device scalar tau
  const float* gu;            // injected uniforms of step t, rows gustride apart ([V] each), or NULL: Philox keyed by ss.coin_state
  int64_t gustride;
};

// -log(u) of the Gumbel uniform u = ((x >> 8) + 0.5) * 2^-24 in (0, 1).  fp32 holds u exactly only below 1/2 (a 24-bit
// significand); above, 1 - u is exact and goes through log1p, so u never rounds to 1 (where the Gumbel noise would be infinite).
__device__ __forceinline__ float neg_log_u24(uint32_t x) {
  const uint32_t m = x >> 8;
  if (m < (1u << 23)) return -logf(((float)m + 0.5f) * (1.0f / 16777216.0f));
  return -log1pf(-(((float)((1u << 24) - 1u - m) + 0.5f) * (1.0f / 16777216.0f)));
}

// Scheduled sampling (lo_decoder_args.ss_prob, lo_tfdec_args.ss_prob), shared by the pointwise LSTM kernels of both decoder
// flavours: the token each row of a 256-thread block of a [nrows][D] launch feeds at this step, chosen and recorded once per row by
// one warp and handed to the row's threads through shared memory.  tok: the teacher tokens (rows tok_stride apart).  Where the coin
// (injected ss.u, else Philox counter (0xFFFFFFFF, t_idx, row0 + r, call)) is below p, the row feeds the lowest-index argmax of
// its ss.prev_logits row (MODE 1) or a Gumbel-max draw from softmax(logits / tau) (MODE 2); ss.prev_logits NULL: the teacher
// token.  Every thread of the block must call it (it synchronises the block); tk_ss receives the token of the thread's row b when
// `live`.
template <int MODE>
__device__ __forceinline__ void ss_block_tokens(const int64_t* __restrict__ tok, int64_t tok_stride, int nrows, int D, int V, int row0,
                                                int t_idx, const SsStep& ss, const GumbelStep& gs, bool live, int b, int64_t& tk_ss) {
  __shared__ int64_t s_tok[256 / 8 + 2];            // rows a 256-thread block touches: <= 256 / D + 1, D % 8 == 0
  const int first = (int)(blockIdx.x * blockDim.x) / D;
  const int last = min(nrows - 1, (int)(blockIdx.x * blockDim.x + blockDim.x - 1) / D);
  const int lane = threadIdx.x & 31;
  for (int r = first + (int)(threadIdx.x >> 5); r <= last; r += (int)(blockDim.x >> 5)) {
    int64_t pick = tok[(int64_t)r * tok_stride];
    if (ss.prev_logits) {
      float u;
      if (ss.u) u = ss.u[(int64_t)r * ss.ustride];
      else {
        const unsigned long long seed = ss.coin_state[0], call = ss.coin_state[1];
        u = u01(philox4x32_10(make_uint4(0xFFFFFFFFu, (uint32_t)t_idx, (uint32_t)(row0 + r), (uint32_t)call),
                              make_uint2((uint32_t)seed, (uint32_t)(seed >> 32))).x);
      }
      if (u < *ss.prob) {                           // warp-uniform
        const float* lg = ss.prev_logits + (int64_t)r * ss.lstride;
        float best = -INFINITY;
        int bi = 0;
        if constexpr (MODE == 2) {
          // Gumbel-max: argmax_v (lg[v] / tau + g_v), g_v = -log(-log u_v), one exact draw from softmax(lg / tau).  Each lane
          // visits its v in increasing order and keeps the first maximum, so the reduction below keeps the lowest index.
          const float tau = *gs.temp;
          if (gs.gu) {
            const float* gu = gs.gu + (int64_t)r * gs.gustride;
            for (int v = lane; v < V; v += 32) {
              const float x = lg[v] / tau - logf(-logf(gu[v]));
              if (x > best) { best = x; bi = v; }
            }
          } else {
            // u_v from word v & 3 of Philox4x32-10(counter = (0x80000000 | v >> 2, t, b, call)): a first counter word neither
            // the dropout stream (j >> 2 < 2^31) nor the coin (0xFFFFFFFF) uses
            const unsigned long long seed = ss.coin_state[0], call = ss.coin_state[1];
            for (int v4 = lane; v4 * 4 < V; v4 += 32) {
              const uint4 w = philox4x32_10(make_uint4(0x80000000u | (uint32_t)v4, (uint32_t)t_idx, (uint32_t)(row0 + r), (uint32_t)call),
                                            make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
              const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
              for (int q = 0; q < 4; q++) {
                const int v = v4 * 4 + q;
                if (v < V) {
                  const float x = lg[v] / tau - logf(neg_log_u24(ws[q]));
                  if (x > best) { best = x; bi = v; }
                }
              }
            }
          }
        } else {
        for (int v = lane; v < V; v += 32) {
          const float x = lg[v];
          if (x > best) { best = x; bi = v; }
        }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best, o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }   // the rule of argmax_kernel (greedy decode)
        }
        pick = bi;
      }
    }
    if (lane == 0) {
      s_tok[r - first] = pick;
      if ((int64_t)r * D >= (int64_t)blockIdx.x * blockDim.x) ss.fed[(int64_t)r * ss.ustride] = pick;   // the block holding j = 0
    }
  }
  __syncthreads();
  if (live) tk_ss = s_tok[b - first];
}

// LSTM cell pointwise (nn.LSTMCell, gate order i,f,g,o).  pre = gtmp + ptab[tok] + hh_pre.
// MODE 0: the token is tok.  MODE 1 / 2 (scheduled sampling): tok is the teacher token; the token fed is chosen here
// (lo_decoder_args.ss_prob, ss_block_tokens) and recorded: the argmax of the previous logits (1) or a Gumbel-max draw from
// softmax(logits / tau) (2).
template <int MODE>
__device__ __forceinline__ void lstm_pw_fwd_body(const float* __restrict__ gtmp, const float* __restrict__ ptab,
                                                 const int64_t* __restrict__ tok, int64_t tok_stride, const float* __restrict__ hh,
                                                 int64_t hh_stride, const float* __restrict__ c_prev, float* __restrict__ gates,
                                                 float* __restrict__ c_out, float* __restrict__ h_out, bf16* __restrict__ h_bf,
                                                 float* __restrict__ hd, int64_t hd_stride, const float* __restrict__ dmask, int nrows,
                                                 int D, int V, const unsigned long long* __restrict__ dstate, float dp, int row0,
                                                 int t_idx, const SsStep& ss, const GumbelStep& gs) {
  constexpr bool SS = MODE != 0;
  // Everything but the gates GEMM result is at least two launches old (token -> table row, the recurrent projection of this step,
  // c_t; the dropout draw depends on nothing): fetched / computed BEFORE griddepcontrol.wait, so only one L2 round trip (gtmp) is left
  // on the critical path of the time loop instead of two dependent ones.
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = idx < nrows * D;
  const int b = live ? idx / D : 0, j = live ? idx % D : 0;
  float a4[4] = {0.f, 0.f, 0.f, 0.f}, cp = 0.f, mult = 1.f;
  int64_t tk_ss = 0;
  // The logits of step t-1 come from the fc GEMM launched right after lstm_pw_fwd_kernel(t-1); the o1 GEMM, the attention and
  // the gates GEMM of step t come in between, so they are three launches old and safe to read before griddepcontrol.wait (as
  // the teacher token is).  The forward keeps that launch order.
  if constexpr (SS) ss_block_tokens<MODE>(tok, tok_stride, nrows, D, V, row0, t_idx, ss, gs, live, b, tk_ss);
  if (live) {
    int64_t tk = SS ? tk_ss : tok[(int64_t)b * tok_stride];
    if (tk < 0) tk = 0;
    if (tk >= V) tk = V - 1;
    const float* pt = ptab + tk * 4 * D;
    const float* h0 = hh + (int64_t)b * hh_stride;
#pragma unroll
    for (int q = 0; q < 4; q++) a4[q] = pt[q * D + j] + h0[q * D + j];
    cp = c_prev[(int64_t)b * D + j];
    if (hd) {
      if (dmask) mult = dmask[(int64_t)b * hd_stride + j];                                           // injected mask (parity tests)
      else if (dstate) mult = philox_dropout_mult(dstate, row0 + b, t_idx, j, dp, 1.f / (1.f - dp));  // drawn here, redrawn in the backward
    }
  }
  pdl_wait();
  pdl_trigger();
  if (!live) return;
  const float* g0 = gtmp + (int64_t)b * 4 * D;
  const float pi = g0[j] + a4[0];
  const float pf = g0[D + j] + a4[1];
  const float pg = g0[2 * D + j] + a4[2];
  const float po = g0[3 * D + j] + a4[3];
  const float i = sigmoidf_(pi), f = sigmoidf_(pf), g = tanhf(pg), o = sigmoidf_(po);
  const float c = f * cp + i * g;
  const float h = o * tanhf(c);
  float* gt = gates + (int64_t)b * 4 * D;
  gt[j] = i; gt[D + j] = f; gt[2 * D + j] = g; gt[3 * D + j] = o;
  c_out[(int64_t)b * D + j] = c;
  h_out[(int64_t)b * D + j] = h;
  if (h_bf) h_bf[(int64_t)b * D + j] = __float2bfloat16_rn(h);
  if (hd) hd[(int64_t)b * hd_stride + j] = h * mult;
  if constexpr (SS) {
    if (ss.hd_bf) ss.hd_bf[(int64_t)b * hd_stride + j] = __float2bfloat16_rn(h * mult);
  }
}

template <bool SS>
__global__ void lstm_pw_fwd_kernel(const float* __restrict__ gtmp, const float* __restrict__ ptab,
                                   const int64_t* __restrict__ tok, int64_t tok_stride, const float* __restrict__ hh,
                                   int64_t hh_stride, const float* __restrict__ c_prev, float* __restrict__ gates,
                                   float* __restrict__ c_out, float* __restrict__ h_out, bf16* __restrict__ h_bf,
                                   float* __restrict__ hd, int64_t hd_stride, const float* __restrict__ dmask, int nrows, int D,
                                   int V, const unsigned long long* __restrict__ dstate, float dp, int row0, int t_idx, SsStep ss) {
  lstm_pw_fwd_body<SS ? 1 : 0>(gtmp, ptab, tok, tok_stride, hh, hh_stride, c_prev, gates, c_out, h_out, h_bf, hd, hd_stride, dmask,
                               nrows, D, V, dstate, dp, row0, t_idx, ss, GumbelStep{});
}
// scheduled sampling with a temperature (lo_decoder_args.ss_temp): the token fed is drawn, not the argmax
__global__ void lstm_pw_fwd_gumbel_kernel(const float* __restrict__ gtmp, const float* __restrict__ ptab,
                                          const int64_t* __restrict__ tok, int64_t tok_stride, const float* __restrict__ hh,
                                          int64_t hh_stride, const float* __restrict__ c_prev, float* __restrict__ gates,
                                          float* __restrict__ c_out, float* __restrict__ h_out, bf16* __restrict__ h_bf,
                                          float* __restrict__ hd, int64_t hd_stride, const float* __restrict__ dmask, int nrows, int D,
                                          int V, const unsigned long long* __restrict__ dstate, float dp, int row0, int t_idx, SsStep ss,
                                          GumbelStep gs) {
  lstm_pw_fwd_body<2>(gtmp, ptab, tok, tok_stride, hh, hh_stride, c_prev, gates, c_out, h_out, h_bf, hd, hd_stride, dmask, nrows, D, V,
                      dstate, dp, row0, t_idx, ss, gs);
}

// backward of the cell pointwise part: dh = dhd[b,t] + dh_next ; writes d(pre-activations), dc_prev in place
__global__ void lstm_pw_bwd_kernel(const float* __restrict__ dhd, int64_t dhd_stride, const float* __restrict__ dmask,
                                   const float* __restrict__ dh_next,
                                   int64_t dhn_stride, float* __restrict__ dc, const float* __restrict__ gates,
                                   const float* __restrict__ c_prev, const float* __restrict__ c_cur,
                                   float* __restrict__ dG, int64_t dG_stride, bf16* __restrict__ dG_bf, float* __restrict__ dxh_zero,
                                   int C, int nrows, int D, const unsigned long long* __restrict__ dstate, float dp, int row0,
                                   int t_idx) {
  // gates / cells come from the forward pass, dhd from the hoisted fc backward, dc from this kernel's previous launch (three launches
  // back), the dropout draw depends on nothing: all fetched before griddepcontrol.wait; only dh_next (the GEMM just before) is after it
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = idx < nrows * D;
  const int b = live ? idx / D : 0, j = live ? idx % D : 0;
  float i = 0.f, f = 0.f, g = 0.f, o = 0.f, tc = 0.f, cpv = 0.f, dhv = 0.f, dcv = 0.f;
  if (live) {
    const float* gt = gates + (int64_t)b * 4 * D;
    i = gt[j]; f = gt[D + j]; g = gt[2 * D + j]; o = gt[3 * D + j];
    tc = tanhf(c_cur[(int64_t)b * D + j]);
    cpv = c_prev[(int64_t)b * D + j];
    dhv = dhd[(int64_t)b * dhd_stride + j];
    if (dmask) dhv *= dmask[(int64_t)b * dhd_stride + j];
    else if (dstate) dhv *= philox_dropout_mult(dstate, row0 + b, t_idx, j, dp, 1.f / (1.f - dp));
    dcv = dc[(int64_t)b * D + j];
  }
  pdl_wait();
  pdl_trigger();
  if (!live) return;
  const float dh = dhv + dh_next[(int64_t)b * dhn_stride + j];
  const float dct = dcv + dh * o * (1.f - tc * tc);
  float* d = dG + (int64_t)b * dG_stride;
  d[j] = dct * g * i * (1.f - i);
  d[D + j] = dct * cpv * f * (1.f - f);
  d[2 * D + j] = dct * i * (1.f - g * g);
  d[3 * D + j] = dh * tc * o * (1.f - o);
  dc[(int64_t)b * D + j] = dct * f;
  if (dG_bf) {
    bf16* q = dG_bf + (int64_t)b * dG_stride;
    q[j] = __float2bfloat16_rn(d[j]);
    q[D + j] = __float2bfloat16_rn(d[D + j]);
    q[2 * D + j] = __float2bfloat16_rn(d[2 * D + j]);
    q[3 * D + j] = __float2bfloat16_rn(d[3 * D + j]);
  }
  if (dxh_zero) {
    // the wgmma split-K GEMMs that follow accumulate with atomics: clear [dgctx | dh] (dh_next was consumed above;
    // entry C+j is this thread's own read location, entries < C are never read here)
    float* z = dxh_zero + (int64_t)b * (C + D);
    z[C + j] = 0.f;
    for (int q = j; q < C; q += D) z[q] = 0.f;
  }
}

// fused cross-entropy forward/backward: warp per (b,t) row.  target = caps[b][t+1]; rows with b >= bt[t] get 0.
__global__ void ce_kernel(const float* __restrict__ logits, const int64_t* __restrict__ caps, int64_t caps_stride,
                          const int32_t* __restrict__ dlen, float* __restrict__ row_loss, float* __restrict__ dlogits,
                          bf16* __restrict__ dlogits_bf, int B, int Tn, int V, int ld, float inv_n) {
  const int row = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= B * Tn) return;
  const int b = row / Tn, t = row % Tn;
  const float* lg = logits + (int64_t)row * ld;
  float* dl = dlogits ? dlogits + (int64_t)row * ld : nullptr;
  bf16* dlb = dlogits_bf ? dlogits_bf + (int64_t)row * ld : nullptr;
  if (t >= dlen[b]) {
    if (lane == 0) row_loss[row] = 0.f;
    if (dl) for (int v = lane; v < ld; v += 32) dl[v] = 0.f;
    if (dlb) for (int v = lane; v < ld; v += 32) dlb[v] = __float2bfloat16_rn(0.f);
    return;
  }
  float mx = -INFINITY;
  for (int v = lane; v < V; v += 32) mx = fmaxf(mx, lg[v]);
  mx = warp_max(mx);
  float se = 0.f;
  for (int v = lane; v < V; v += 32) se += expf(lg[v] - mx);
  se = warp_sum(se);
  const float lse = mx + logf(se);
  int64_t tg = caps[(int64_t)b * caps_stride + t + 1];
  if (tg < 0) tg = 0;
  if (tg >= V) tg = V - 1;
  if (lane == 0) row_loss[row] = lse - lg[tg];
  if (dl)
    for (int v = lane; v < ld; v += 32) {
      const float g = v < V ? (expf(lg[v] - lse) - (v == (int)tg ? 1.f : 0.f)) * inv_n : 0.f;
      dl[v] = g;
      if (dlb) dlb[v] = __float2bfloat16_rn(g);
    }
}

// generic backward: dlogits (+ bf16 mirror) = the caller's d predictions, source rows (b, t) batch-major; rows with t >= dlen[b]
// (dlen NULL: none) and columns [V, ld) get zeros (same rule as ce_kernel).  Destination row: the same (b * Tn + t), or with
// tm_B > 0 the time-major t * tm_B + b (TF flavour).  grid (ld / 128 blocks, up to nrows rows; y strides over the rest)
__global__ void dpred_kernel(const float* __restrict__ dpred, int64_t dpred_stride, const int32_t* __restrict__ dlen,
                             float* __restrict__ dlogits, bf16* __restrict__ dlogits_bf, int Tn, int V, int ld, int64_t nrows,
                             int tm_B) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= ld) return;
  for (int64_t row = blockIdx.y; row < nrows; row += gridDim.y) {
    const int b = (int)(row / Tn), t = (int)(row % Tn);
    const float g = (v < V && (!dlen || t < dlen[b])) ? dpred[row * dpred_stride + v] : 0.f;
    const int64_t drow = tm_B > 0 ? (int64_t)t * tm_B + b : row;
    dlogits[drow * ld + v] = g;
    if (dlogits_bf) dlogits_bf[drow * ld + v] = __float2bfloat16_rn(g);
  }
}

// doubly-stochastic regulariser: S = sum_t alpha ; sq -> row_loss tail ; dreg = -2 alpha_c (1-S)/(B R)
__global__ void reg_kernel(const float* __restrict__ alphas, float* __restrict__ sq, float* __restrict__ dreg, int B, int Tn,
                           int R, float alpha_c) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * R) return;
  const int b = idx / R, r = idx % R;
  float S = 0.f;
  for (int t = 0; t < Tn; t++) S += alphas[((int64_t)b * Tn + t) * R + r];
  const float d = 1.f - S;
  sq[idx] = d * d;
  if (dreg) dreg[idx] = -2.f * alpha_c * d / ((float)B * (float)R);
}

// sreg[b,t] = sum_r alpha[b,t,r] dreg[b,r]  (warp per (b,t))
__global__ void sreg_kernel(const float* __restrict__ alphas, const float* __restrict__ dreg, int64_t dreg_bstride,
                            int64_t dreg_tstride, float* __restrict__ sreg, int B, int Tn, int R) {
  const int row = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= B * Tn) return;
  const int b = row / Tn, t = row % Tn;
  float s = 0.f;
  for (int r = lane; r < R; r += 32)
    s = fmaf(alphas[(int64_t)row * R + r], dreg[(int64_t)b * dreg_bstride + (int64_t)t * dreg_tstride + r], s);
  s = warp_sum(s);
  if (lane == 0) sreg[row] = s;
}

// deterministic final reduction: loss[0]=total, [1]=ce, [2]=reg, [3]=n_valid
__global__ void loss_finalize_kernel(const float* __restrict__ row_loss, int n_rows, const float* __restrict__ sq, int n_sq,
                                     float inv_n, float alpha_c, float* __restrict__ loss) {
  __shared__ float red[2][32];
  float a = 0.f, c = 0.f;
  for (int i = threadIdx.x; i < n_rows; i += blockDim.x) a += row_loss[i];
  for (int i = threadIdx.x; i < n_sq; i += blockDim.x) c += sq[i];
  a = warp_sum(a);
  c = warp_sum(c);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float ta = 0.f, tcq = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) { ta += red[0][w]; tcq += red[1][w]; }
    const float ce = ta * inv_n, reg = n_sq ? tcq / (float)n_sq : 0.f;
    loss[0] = ce + alpha_c * reg;
    loss[1] = ce;
    loss[2] = reg;
    loss[3] = 1.f / inv_n;
  }
}

// dptab[v][:] = sum over (t,b) with caps[b][t] == v (and t < dlen[b]) of dG[t][b][:]   (deterministic order)
__global__ void dptab_kernel(const float* __restrict__ dcat, int64_t row_stride, int64_t step_stride, int col0,
                             const int64_t* __restrict__ caps, int64_t caps_stride, const int32_t* __restrict__ dlen,
                             float* __restrict__ dptab, int B, int Tn, int G) {
  const int v = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ unsigned s_bits[8];
  float acc = 0.f;
  const int total = B * Tn;
  for (int base = 0; base < total; base += 256) {
    const int idx = base + threadIdx.x;
    bool hit = false;
    if (idx < total) {
      const int b = idx / Tn, t = idx % Tn;
      hit = (t < dlen[b]) && (caps[(int64_t)b * caps_stride + t] == (int64_t)v);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0) s_bits[threadIdx.x >> 5] = bal;
    __syncthreads();
    if (j < G) {
#pragma unroll
      for (int w = 0; w < 8; w++) {
        unsigned bits = s_bits[w];
        while (bits) {                                  // ascending index order -> deterministic sum
          const int k = __ffs(bits) - 1;
          bits &= bits - 1;
          const int id = base + w * 32 + k;
          const int b = id / Tn, t = id % Tn;
          acc += dcat[(int64_t)t * step_stride + (int64_t)b * row_stride + col0 + j];
        }
      }
    }
    __syncthreads();
  }
  if (j < G) dptab[(int64_t)v * G + j] = acc;
}

// one-hot rows (t,b) x Vp for the tensor-core form of the embedding-table gradient: dptab = onehot^T @ dG
__global__ void onehot_kernel(const int64_t* __restrict__ caps, int64_t caps_stride, const int32_t* __restrict__ dlen,
                              bf16* __restrict__ oh, int B, int Tn, int Vp) {
  const int64_t total = (int64_t)B * Tn * Vp;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % Vp);
    const int64_t row = i / Vp;
    const int b = (int)(row % B), t = (int)(row / B);
    const bool hit = (t < dlen[b]) && (caps[(int64_t)b * caps_stride + t] == (int64_t)v);
    oh[i] = __float2bfloat16_rn(hit ? 1.f : 0.f);
  }
}

// bf16 operands of the batched tensor-core GEMM d enc[b] += alphas[b]^T dctx[:, b, :]:
//   alphas fp32 [B*T][R] -> bf16 [B*T][Rp] (rows padded to a multiple of 8 elements = 16 bytes, a TMA stride requirement)
__global__ void cast_pad_rows_kernel(const float* __restrict__ x, bf16* __restrict__ y, int64_t rows, int R, int Rp) {
  const int64_t total = rows * Rp;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / Rp;
    const int c = (int)(i % Rp);
    y[i] = __float2bfloat16_rn(c < R ? x[r * R + c] : 0.f);
  }
}
//   dctx fp32 [T][B][C] -> bf16 [B][T][C]
__global__ void cast_tb_to_bt_kernel(const float* __restrict__ x, bf16* __restrict__ y, int T, int B, int C) {
  const int64_t total = (int64_t)T * B * (C / 8);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % (C / 8));
    const int64_t tb = i / (C / 8);
    const int b = (int)(tb % B), t = (int)(tb / B);
    float v[8];
    ld8(x + tb * C + c8 * 8, v);
    st8(y + ((int64_t)b * T + t) * C + c8 * 8, v);
  }
}

// denc[b][r][:] += dmean[b][:] / R
__global__ void add_rowbcast_kernel(float* __restrict__ denc, const float* __restrict__ dmean, int R, int C, float scale,
                                    int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t b = i / ((int64_t)R * C);
    denc[i] += dmean[b * C + c] * scale;
  }
}

// denc[b][r][c] += alpha[b][r] * dctx[b][c]   (the context read of one attention step, seq2seq_torch.py:190)
__global__ void add_outer_kernel(float* __restrict__ denc, const float* __restrict__ alpha, const float* __restrict__ dctx, int R, int C,
                                 int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t br = i / C;
    denc[i] = fmaf(alpha[br], dctx[(br / R) * C + c], denc[i]);
  }
}

// out[n][k] = in[k][n]  (in [K][ld_in] -> out [N][ld_out]), generic small transpose with dtype
template <typename T>
__global__ void transpose_kernel(const T* __restrict__ in, int64_t ld_in, T* __restrict__ out, int64_t ld_out, int K, int N) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += 8)
    if (k0 + i < K && n0 + threadIdx.x < N) tile[i][threadIdx.x] = ldf(in + (int64_t)(k0 + i) * ld_in + n0 + threadIdx.x);
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8)
    if (n0 + i < N && k0 + threadIdx.x < K) stf(out + (int64_t)(n0 + i) * ld_out + k0 + threadIdx.x, tile[threadIdx.x][i]);
}

__global__ void argmax_kernel(const float* __restrict__ logits, int V, int64_t* __restrict__ tokens, int64_t tok_stride,
                              int64_t* __restrict__ next_tok, int32_t* __restrict__ finished, int64_t end_id, int B) {
  const int b = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  float best = -INFINITY;
  int bi = 0;
  for (int v = lane; v < V; v += 32) {
    const float x = logits[(int64_t)b * V + v];
    if (x > best) { best = x; bi = v; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }   // lowest index wins ties (torch.argmax)
  }
  if (lane == 0) {
    tokens[(int64_t)b * tok_stride] = bi;
    next_tok[b] = bi;
    if (bi == end_id) finished[b] = 1;
  }
}


// ------------------------------------------------------------------------------------------------
// beam search step (beam_search_decoder_cell.py:123-187): one block per image.
//   lp = log_softmax(logits) ; finished beams -> [END: 0, else: dtype.min] ; total = prev + lp ;
//   time 0: beam 0 only ; top-k(beam) over beam*V (lower flat index wins ties) ; id = idx % V ; parent = idx / V
// ------------------------------------------------------------------------------------------------
#define LO_BEAM_MAX 16
__global__ void __launch_bounds__(256) beam_step_kernel(const float* __restrict__ logits, int V, int beam, int t, int64_t end_id,
                                                        float* __restrict__ logp, int32_t* __restrict__ finished,
                                                        int64_t* __restrict__ ids, int64_t* __restrict__ parents,
                                                        int32_t* __restrict__ fin_hist, int64_t* __restrict__ next_tok,
                                                        int32_t* __restrict__ parent_rows, int max_steps, float div_log_gamma,
                                                        float div_prob, const float* __restrict__ div_u,
                                                        const unsigned long long* __restrict__ div_state) {
  extern __shared__ float s_tot[];            // [beam*V] (+ [beam*V] penalties when the diversity penalty is on)
  __shared__ float s_red[8];
  __shared__ int s_redi[8];
  __shared__ float s_lse[LO_BEAM_MAX];
  __shared__ float s_newp[LO_BEAM_MAX];
  __shared__ int s_newi[LO_BEAM_MAX];
  const int img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int row0 = img * beam;
  // log-sum-exp per beam row (warp w handles rows w, w+8, ...)
  for (int k = wid; k < beam; k += 8) {
    const float* lg = logits + (int64_t)(row0 + k) * V;
    float mx = -INFINITY;
    for (int v = lane; v < V; v += 32) mx = fmaxf(mx, lg[v]);
    mx = warp_max(mx);
    float se = 0.f;
    for (int v = lane; v < V; v += 32) se += expf(lg[v] - mx);
    se = warp_sum(se);
    if (lane == 0) s_lse[k] = mx + logf(se);
  }
  __syncthreads();
  const int nb = (t == 0) ? 1 : beam;          // beam_search_decoder_cell.py:159-160
  const int total = nb * V;
  for (int i = tid; i < total; i += 256) {
    const int k = i / V, v = i % V;
    float lp = logits[(int64_t)(row0 + k) * V + v] - s_lse[k];
    if (finished[row0 + k]) lp = (v == (int)end_id) ? 0.f : -3.4028234663852886e38f;   // mask_probs :353-367
    s_tot[i] = logp[row0 + k] + lp;
  }
  __syncthreads();
  if (div_log_gamma != 0.f && div_prob > 0.f) {
    // add_div_penalty (beam_search_decoder_cell.py:258-287, Li et al. 2016): rank of every candidate inside its beam row
    // (0 = best; tf.nn.top_k(sorted) puts the lower index first among equals), penalty = log(gamma) * rank, applied where
    // div_prob > u with u ~ U[0,1) per (image, beam, token) — injected (div_u, parity tests) or drawn from Philox
    float* s_pen = s_tot + beam * V;
    for (int i = tid; i < total; i += 256) {
      const int k = i / V, v = i % V;
      const float x = s_tot[i];
      const float* rowp = s_tot + k * V;
      int rank = 0;
      for (int q = 0; q < V; q++) {
        const float y = rowp[q];
        rank += (y > x || (y == x && q < v)) ? 1 : 0;
      }
      float u;
      if (div_u) u = div_u[(int64_t)(row0 + k) * V + v];
      else {
        const uint4 r = philox4x32_10(make_uint4((uint32_t)(v >> 2), (uint32_t)t, (uint32_t)(row0 + k), (uint32_t)div_state[1]),
                                      make_uint2((uint32_t)div_state[0], (uint32_t)(div_state[0] >> 32)));
        u = u01((v & 3) == 0 ? r.x : ((v & 3) == 1 ? r.y : ((v & 3) == 2 ? r.z : r.w)));
      }
      s_pen[i] = div_prob > u ? div_log_gamma * (float)rank : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < total; i += 256) s_tot[i] += s_pen[i];
    __syncthreads();
  }
  for (int j = 0; j < beam; j++) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < total; i += 256) {
      const float x = s_tot[i];
      if (x > best || (x == best && i < bi)) { best = x; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) { s_red[wid] = best; s_redi[wid] = bi; }
    __syncthreads();
    if (tid == 0) {
      float b2 = s_red[0];
      int i2 = s_redi[0];
      for (int w = 1; w < 8; w++)
        if (s_red[w] > b2 || (s_red[w] == b2 && s_redi[w] < i2)) { b2 = s_red[w]; i2 = s_redi[w]; }
      if (i2 == 0x7fffffff) i2 = 0;          // fewer candidates than beams (beam*V < beam): cannot happen for V >= beam
      s_newp[j] = b2;
      s_newi[j] = i2;
      s_tot[i2] = -INFINITY;                  // remove from the candidate set
    }
    __syncthreads();
  }
  if (tid < beam) {
    const int idx = s_newi[tid];
    const int id = idx % V, par = idx / V;
    const int fin = finished[row0 + par] | (id == (int)end_id ? 1 : 0);
    const int64_t o = ((int64_t)img * max_steps + t) * beam + tid;
    ids[o] = id;
    parents[o] = par;
    fin_hist[o] = fin;
    next_tok[row0 + tid] = id;
    parent_rows[row0 + tid] = row0 + par;
    logp[row0 + tid] = s_newp[tid];           // (every read of the old logp happened before the top-k loop)
  }
  __syncthreads();                            // finished[] of the parents is read above, overwritten below
  if (tid < beam) {
    const int64_t o = ((int64_t)img * max_steps + t) * beam + tid;
    finished[row0 + tid] = fin_hist[o];
  }
}

// dst[r][:] = src[rows[r]][:] (+ bf16 mirror of dst)  (state gather by parents, gather_helper beam_search_decoder_cell.py:370-391)
__global__ void gather_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ rows, float* __restrict__ dst,
                                   bf16* __restrict__ dst_bf, int n, int W) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * W) return;
  const int r = idx / W, j = idx % W;
  const float v = src[(int64_t)rows[r] * W + j];
  dst[idx] = v;
  if (dst_bf) dst_bf[idx] = __float2bfloat16_rn(v);
}

__global__ void fin_hist_kernel(const int32_t* __restrict__ finished, int32_t* __restrict__ hist, int64_t stride, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) hist[(int64_t)i * stride] = finished[i];
}

__global__ void fill_i64_kernel(int64_t* p, int64_t v, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

__global__ void bump_counter_kernel(unsigned long long* c) { *c += 1ull; }

__global__ void dlen_kernel(int32_t* dlen, int B, int Tn, int full) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) dlen[i] = full;
  (void)Tn;
}

// ------------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------------
struct Dims {
  int B, T, R, C, A, D, E, V, O1, G, Vl;
};
static inline Dims dims(const lo_decoder_args* a) {
  return Dims{a->B, a->T, a->R, a->C, a->A, a->D, a->E, a->V, a->A + a->C + 4 * a->D, 4 * a->D, a->ldl > 0 ? a->ldl : a->V};
}

// bf16 staging used when impl == TC: mirrors written by the step kernels feed the wgmma GEMMs directly
struct BfViews {
  bool on;
  bf16 *dcat, *hall, *gctx, *wet, *onehot, *hd, *dlogits, *wfct, *alphas, *dctx, *dptab, *wihT;
};
static inline int64_t rpad8(int64_t r) { return (r + 7) / 8 * 8; }
static BfViews bf_views(const lo_decoder_args* a, const Dims& d) {
  BfViews v{false, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  if (a->impl == LO_IMPL_TC && a->dt == LO_BF16 && a->bfwork && tc_available()) {
    const int64_t TB = (int64_t)d.T * d.B;
    v.on = true;
    v.dcat = (bf16*)a->bfwork;
    v.hall = v.dcat + TB * d.O1;
    v.gctx = v.hall + (TB + d.B) * d.D;
    v.wet = v.gctx + TB * d.C;
    v.onehot = v.wet + (int64_t)d.A * d.C;
    v.hd = v.onehot + TB * ((d.V + 7) / 8 * 8);
    v.dlogits = v.hd + TB * d.D;
    v.wfct = v.dlogits + TB * d.Vl;
    v.alphas = v.wfct + (int64_t)d.D * d.Vl;               // [B][T][roundup8(R)] (zero padded): A operand of the batched alpha^T dctx GEMM
    v.dctx = v.alphas + TB * rpad8(d.R);                   // [B][T][C]
    v.dptab = v.dctx + TB * d.C;                           // [V][4D] bf16 copy of the embedding-table gradient
    v.wihT = v.dptab + (int64_t)d.V * d.G;                 // [E][4D] = (weight_ih[:, :E])^T
  }
  return v;
}

static int check_args(const lo_decoder_args* a) {
  LO_CHECK_ARG(a != nullptr, "args");
  LO_CHECK_ARG(a->B > 0 && a->T > 0 && a->R > 0 && a->V > 1, "B,T,R,V");
  LO_CHECK_ARG(a->A == a->C && (a->C == 256 || a->C == 512 || a->C == 1024), "attention_dim == encoder_dim in {256,512,1024}");
  LO_CHECK_ARG(a->D % 8 == 0 && a->E % 8 == 0, "D, E multiples of 8");
  LO_CHECK_ARG(a->dt == LO_F32 || a->dt == LO_BF16, "dt");
  LO_CHECK_ARG(a->ldl == 0 || a->ldl >= a->V, "ldl >= V");
  LO_CHECK_ARG(a->rows_per_img <= 1 || a->B % a->rows_per_img == 0, "B must be a multiple of rows_per_img");
  LO_CHECK_ARG(a->phase >= 0 && a->phase <= 2, "phase in 0..2");
  LO_CHECK_ARG(a->bt_host && a->caps && a->enc && a->work, "null pointer");
  LO_CHECK_ARG(a->has_dropout != 2 || (a->dropout_state && a->dropout_p >= 0.f && a->dropout_p < 1.f),
               "has_dropout=2 needs dropout_state, 0 <= dropout_p < 1");
  if (a->ss_prob) {
    LO_CHECK_ARG(a->fed, "scheduled sampling (ss_prob) needs fed");
    LO_CHECK_ARG(a->ss_u || a->dropout_state, "scheduled sampling (ss_prob) needs ss_u or dropout_state for its coin");
    LO_CHECK_ARG(a->phase == 0, "scheduled sampling (ss_prob) needs phase 0: no per-step head when a layer sits between h and fc");
    LO_CHECK_ARG(a->rows_per_img <= 1, "scheduled sampling (ss_prob) needs rows_per_img <= 1");
    LO_CHECK_ARG(!a->ss_gu || a->ss_temp, "ss_gu (injected Gumbel uniforms) needs ss_temp");
  } else {
    LO_CHECK_ARG(!a->ss_temp && !a->ss_gu, "ss_temp / ss_gu (sampling with a temperature) need ss_prob");
  }
  for (int t = 0; t < a->T; t++) {
    LO_CHECK_ARG(a->bt_host[t] >= 1 && a->bt_host[t] <= a->B, "bt_host out of range");
    if (t) LO_CHECK_ARG(a->bt_host[t] <= a->bt_host[t - 1], "bt_host must be non-increasing");
  }
  return LO_OK;
}

// per-image region counts (reg_off / reg_off_host of lo_decoder_args and lo_tfdec_args): decode entry points only.  `decode`: the
// call is a greedy / beam entry point (the offsets are validated), otherwise a training one (the offsets are refused).
static int check_reg_off(const int32_t* reg_off, const int32_t* reg_off_host, int B, int rows_per_img, int R, bool decode) {
  if (!reg_off && !reg_off_host) return LO_OK;
  LO_CHECK_ARG(decode, "reg_off / reg_off_host (per-image region counts) are for the decode entry points only");
  LO_CHECK_ARG(reg_off && reg_off_host, "reg_off and reg_off_host must be set together");
  LO_CHECK_ARG(g_opt_att_pipe, "per-image region counts (reg_off) need the pipelined attention kernels (att_pipe = 1)");
  const int rpi = rows_per_img > 1 ? rows_per_img : 1;
  LO_CHECK_ARG(reg_off_host[0] == 0, "reg_off_host[0] must be 0");
  for (int i = 0; i < B / rpi; i++) {
    const int n = reg_off_host[i + 1] - reg_off_host[i];
    LO_CHECK_ARG(n >= 1 && n <= R, "region count of every image in 1..R (reg_off_host)");
  }
  return LO_OK;
}
template <class Args>            // lo_decoder_args or lo_tfdec_args
static int check_reg_off(const Args* a, bool decode) {
  return check_reg_off(a->reg_off, a->reg_off_host, a->B, a->rows_per_img, a->R, decode);
}
// the ragged attention state of a decode call: map in the second attention region of `work` (the time loop's launches use the first)
static AttRagged ragged_of(const lo_decoder_args* a) {
  return AttRagged{a->reg_off, a->reg_off_host, (char*)a->work + lo_attention_workspace_bytes(a->B, a->C), 0};
}

static int* work_counters(const lo_decoder_args* a) { return (int*)a->work; }
// ReLU mask bits of step t (NULL when the scheme is off)
static inline uint8_t* att_mask_at(const lo_decoder_args* a, int t) {
  if (!a->att_mask || !g_opt_att_maskbits || !g_opt_att_pipe || a->rows_per_img > 1) return nullptr;
  return a->att_mask + (int64_t)t * a->B * ((a->R + 1) & ~1) * (a->A / 8);      // rows padded to an even count (pair layout)
}
static float* work_partials(const lo_decoder_args* a) { return (float*)((char*)a->work + att_partials_offset(a->B)); }
static int32_t* work_dlen(const lo_decoder_args* a) { return (int32_t*)((char*)a->work + 2048); }

static int attention_forward_launch(const void* att1, const void* enc, int dt, const float* att2, int64_t att2_stride,
                                    const float* wf, float* alpha, int64_t alpha_stride, float* ctx, float* gate_pre,
                                    int64_t gate_stride, float* gctx, bf16* gctx_bf, int B, int R, int C, void* work, cudaStream_t st,
                                    int rpi = 1, uint8_t* mask_out = nullptr, int abi = 0) {
  if (rpi < 1) rpi = 1;
  if (g_opt_att_pipe) {
    AttFwdArgs x{att1, enc, att2, att2_stride, wf, alpha, alpha_stride, ctx, gate_pre, gate_stride, gctx, gctx_bf, B, R, work, rpi,
                 0, 0, mask_out, abi};
    return attention_fwd_pipe(x, dt, C, st);
  }
  const int ns = att_splits(B);
  int* cnt = (int*)work;
  float* part = (float*)((char*)work + att_partials_offset(B));
  dim3 grid(ns, B);
#define LO_ATT_FWD(T, NV)                                                                                           \
  attention_fwd_kernel<T, NV><<<grid, LO_ATT_THREADS, 0, st>>>((const T*)att1, (const T*)enc, att2, att2_stride, wf, \
                                                               alpha, alpha_stride, ctx, gate_pre, gate_stride, gctx, gctx_bf, R, ns, cnt, part, rpi)
  if (dt == LO_F32) {
    if (C == 256) LO_ATT_FWD(float, 1); else if (C == 512) LO_ATT_FWD(float, 2); else LO_ATT_FWD(float, 4);
  } else {
    if (C == 256) LO_ATT_FWD(bf16, 1); else if (C == 512) LO_ATT_FWD(bf16, 2); else LO_ATT_FWD(bf16, 4);
  }
#undef LO_ATT_FWD
  LO_LAUNCH_OK();
  return LO_OK;
}

// builds dlen[b] (device) = number of steps row b decodes, from the host bt[] array, via tiny memcpy-free kernels
static int upload_dlen(const lo_decoder_args* a, cudaStream_t st) {
  // dlen[b] = #{t : bt[t] > b}.  bt is non-increasing, so rows [bt[t], bt[t-1]) have dlen = t.
  int32_t* dl = work_dlen(a);
  LO_CHECK_ARG(a->B <= 512, "B <= 512 (dlen scratch)");
  LO_CUDA(cudaMemsetAsync(dl, 0, (size_t)a->B * 4, st));   // rows that never decode (caption length 1)
  // rows below bt[T-1] decode all T steps
  dlen_kernel<<<cdiv(a->B, 128), 128, 0, st>>>(dl, a->bt_host[a->T - 1], a->T, a->T);
  LO_LAUNCH_OK();
  for (int t = a->T - 1; t >= 1; t--) {
    const int lo_ = a->bt_host[t], hi_ = a->bt_host[t - 1];
    if (hi_ > lo_) {
      dlen_kernel<<<cdiv(hi_ - lo_, 128), 128, 0, st>>>(dl + lo_, hi_ - lo_, a->T, t);
      LO_LAUNCH_OK();
    }
  }
  return LO_OK;
}

// x = hi + lo with hi = bf16(x), lo = bf16(x - hi): two bf16 GEMMs then reproduce an fp32-input GEMM to ~2^-17 relative
__global__ void split_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ hi, bf16* __restrict__ lo, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    const bf16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

static int forward_prologue(const lo_decoder_args* a, const Dims& d, cudaStream_t st) {
  const int dt = a->dt;
  const int rpi = a->rows_per_img > 1 ? a->rows_per_img : 1;
  // att1 = enc @ W_e^T + b_e   (hoisted: the reference recomputes it every step, seq2seq_torch.py:186); packed layout: every region
  // of every image once
  const int enc_rows = a->reg_off_host ? a->reg_off_host[d.B / rpi] : (d.B / rpi) * d.R;
  LO_TRY(gemm_nt(a->enc, dt, d.C, a->w_enc_att, dt, d.C, a->att1, dt, d.A, enc_rows, d.A, d.C, a->b_enc_att, 0, 0, a->impl, st));
  const BfViews bv0 = bf_views(a, d);
  // embedding -> gate projection table (replaces embedding lookup + x[:, :E] @ W_ih[:, :E]^T, seq2seq_torch.py:291,:313)
  if (bv0.on && d.E % 64 == 0) {
    LO_TRY(tc_gemm_nt_ex((const bf16*)a->emb, d.E, (const bf16*)a->w_ih, d.E + d.C, a->ptab, LO_F32, d.G, d.V, d.G, d.E, a->b_ih, 0, 0, 1,
                         0, 0, st));
  } else {
    LO_TRY(gemm_nt(a->emb, dt, d.E, a->w_ih, dt, d.E + d.C, a->ptab, LO_F32, d.G, d.V, d.G, d.E, a->b_ih, 0, 0, LO_IMPL_SIMT, st));
  }
  // init_hidden_state (seq2seq_torch.py:255-265)
  {
    dim3 grid(cdiv(d.C, 256), d.B);
    if (a->reg_off)
      LO_DISPATCH_DT(dt, T, (mean_segments_kernel<T><<<grid, 256, 0, st>>>((const T*)a->enc, a->mean, a->reg_off, d.C, rpi)));
    else
      LO_DISPATCH_DT(dt, T, (mean_rows_kernel<T><<<grid, 256, 0, st>>>((const T*)a->enc, a->mean, d.R, d.C, rpi)));
    LO_LAUNCH_OK();
  }
  const size_t es = dt == LO_F32 ? 4 : 2;
  if (bv0.on && d.C % 64 == 0 && d.T >= 2) {
    // the row means stay fp32-accurate: hi/lo bf16 split (staged in the not-yet-used gctx mirrors of steps 0 and 1)
    bf16* mean_hi = bv0.gctx;
    bf16* mean_lo = bv0.gctx + (int64_t)d.B * d.C;
    split_bf16_kernel<<<cdiv((long)d.B * d.C, 256), 256, 0, st>>>(a->mean, mean_hi, mean_lo, (int64_t)d.B * d.C);
    LO_LAUNCH_OK();
    const bf16* w_h = (const bf16*)a->w_init;
    const bf16* w_c = w_h + (int64_t)d.D * d.C;
    LO_TRY(tc_gemm_nt_ex(mean_hi, d.C, w_h, d.C, a->hall, LO_F32, d.D, d.B, d.D, d.C, a->b_init, 0, 0, 1, 0, 1, st));
    LO_TRY(tc_gemm_nt_ex(mean_lo, d.C, w_h, d.C, a->hall, LO_F32, d.D, d.B, d.D, d.C, nullptr, 1, 0, 1, 0, 1, st));
    LO_TRY(tc_gemm_nt_ex(mean_hi, d.C, w_c, d.C, a->call, LO_F32, d.D, d.B, d.D, d.C, a->b_init + d.D, 0, 0, 1, 0, 1, st));
    LO_TRY(tc_gemm_nt_ex(mean_lo, d.C, w_c, d.C, a->call, LO_F32, d.D, d.B, d.D, d.C, nullptr, 1, 0, 1, 0, 1, st));
  } else {
    LO_TRY(gemm_nt(a->mean, LO_F32, d.C, a->w_init, dt, d.C, a->hall, LO_F32, d.D, d.B, d.D, d.C, a->b_init, 0, 0, LO_IMPL_SIMT, st));
    LO_TRY(gemm_nt(a->mean, LO_F32, d.C, (const char*)a->w_init + (size_t)d.D * d.C * es, dt, d.C, a->call, LO_F32, d.D, d.B,
                   d.D, d.C, a->b_init + d.D, 0, 0, LO_IMPL_SIMT, st));
  }
  const BfViews bv = bf_views(a, d);
  if (bv.on) LO_TRY(lo_cast(a->hall, LO_F32, bv.hall, LO_BF16, (int64_t)d.B * d.D, (void*)st));
  return LO_OK;
}

// C (+)= A W^T for the per-step GEMMs of the time loops (M <= B rows): the mma.sync kernel for <= 64 rows of the bf16 mirror Abf,
// wgmma above, CUDA cores on the fp32 operand A32 when there are no mirrors (tc false).  The tensor-core paths run `splits` K slices
// (atomic_acc: added onto C with fp32 atomics); the CUDA-core path writes C or, with `acc`, adds to it.  Option "deterministic" on
// wgmma: one K slice, so every element of C receives a single atomic add onto its base value and the result does not depend on the
// order in which CTAs finish (the mma.sync kernel orders its slices itself).
static int step_gemm_nt(bool tc, const float* A32, const bf16* Abf, int64_t lda, const void* W, int dtW, int64_t ldw, float* C,
                        int64_t ldc, int M, int N, int K, const float* bias, int acc, int splits, int atomic_acc, cudaStream_t st) {
  if (tc && g_opt_skinny_mma && M <= 64) return skinny_gemm_nt(Abf, lda, (const bf16*)W, ldw, C, ldc, M, N, K, bias, splits, atomic_acc, st);
  if (tc)
    return tc_gemm_nt_ex(Abf, lda, (const bf16*)W, ldw, C, LO_F32, ldc, M, N, K, bias, 0, 0, g_opt_det ? 1 : splits, atomic_acc, 1, st);
  return gemm_nt(A32, LO_F32, lda, W, dtW, ldw, C, LO_F32, ldc, M, N, K, bias, acc, 0, LO_IMPL_SIMT, st);
}

// logits = fc(h) for M rows inside a time loop (sampling head, greedy and beam decode): the dispatcher's mma.sync kernel for <= 64
// rows of the bf16 mirror hbf, CUDA cores on h32 otherwise
static int head_nt(const lo_decoder_args* a, bool tc, const float* h32, const bf16* hbf, int64_t ldh, float* logits, int64_t ldl, int M,
                   cudaStream_t st) {
  if (tc) return gemm_nt(hbf, LO_BF16, ldh, a->w_fc, LO_BF16, a->D, logits, LO_F32, ldl, M, a->V, a->D, a->b_fc, 0, 0, LO_IMPL_TC, st);
  return gemm_nt(h32, LO_F32, ldh, a->w_fc, a->dt, a->D, logits, LO_F32, ldl, M, a->V, a->D, a->b_fc, 0, 0, LO_IMPL_SIMT, st);
}

// one decoder step t for the first nrows rows of the batch (those still decoding); rg: decode with per-image region counts (the
// whole batch), else null; tok: token ids consumed at this step
static int forward_step(const lo_decoder_args* a, const Dims& d, int t, int nrows, const AttRagged* rg, const int64_t* tok,
                        int64_t tok_stride, float* hd_t, int64_t hd_stride, const float* dmask_t, cudaStream_t st) {
  const int dt = a->dt;
  const bool sampling = a->ss_prob && hd_t;     // scheduled sampling: token chosen in the cell, head inside the loop
  const size_t es = dt == LO_F32 ? 4 : 2;
  const int64_t cur = (int64_t)t * d.B, nxt = (int64_t)(t + 1) * d.B;     // first row of steps t and t + 1 (time-major arrays)
  float* o1 = a->out1 + cur * d.O1;
  // [att2 | gate_pre | hh_pre] = h_prev @ [W_d; W_beta; W_hh]^T + b   (seq2seq_torch.py:187, :311, LSTMCell hh part)
  const BfViews bv = bf_views(a, d);
  if (!(g_opt_dbg_skip & 4))
    LO_TRY(step_gemm_nt(bv.on, a->hall + cur * d.D, bv.on ? bv.hall + cur * d.D : nullptr, d.D, a->wcat1, dt, d.D, o1, d.O1, nrows,
                        d.O1, d.D, a->bcat1, 0, 1, 0, st));
  if (rg) {
    if (!(g_opt_dbg_skip & 2)) {
      AttFwdArgs x{a->att1, a->enc, o1, d.O1, a->w_full, a->alphas + t * d.R, (int64_t)d.T * d.R, a->ctx + cur * d.C, o1 + d.A,
                   d.O1, a->gctx + cur * d.C, bv.on ? bv.gctx + cur * d.C : nullptr, nrows, d.R, a->work, a->rows_per_img, 0, 0, nullptr, 0};
      LO_TRY(attention_fwd_ragged(x, *rg, dt, d.C, st));
    }
  } else if (!(g_opt_dbg_skip & 2))
  LO_TRY(attention_forward_launch(a->att1, a->enc, dt, o1, d.O1, a->w_full, a->alphas + t * d.R, (int64_t)d.T * d.R, a->ctx + cur * d.C,
                                  o1 + d.A, d.O1, a->gctx + cur * d.C, bv.on ? bv.gctx + cur * d.C : nullptr, nrows, d.R, d.C, a->work, st,
                                  a->rows_per_img, hd_t ? att_mask_at(a, t) : nullptr));
  if (g_opt_dbg_skip & 4) return LO_OK;
  // gates_x = (gate*ctx) @ W_ih[:, E:]^T
  LO_TRY(step_gemm_nt(bv.on, a->gctx + cur * d.C, bv.on ? bv.gctx + cur * d.C : nullptr, d.C, (const char*)a->w_ih + (size_t)d.E * es, dt,
                      d.E + d.C, a->gtmp, d.G, nrows, d.G, d.C, nullptr, 0, 1, 0, st));
  SsStep ss{};
  if (sampling) {
    ss.prev_logits = t > 0 ? a->logits + (int64_t)(t - 1) * d.Vl : nullptr;
    ss.lstride = (int64_t)d.T * d.Vl;
    ss.prob = a->ss_prob;
    ss.u = a->ss_u ? a->ss_u + t : nullptr;
    ss.coin_state = (const unsigned long long*)a->dropout_state;
    ss.ustride = d.T;
    ss.fed = a->fed + t;
    ss.hd_bf = bv.on ? bv.hd + t * d.D : nullptr;
  }
  // the pointwise launch; `extra` is the GumbelStep of the sampling kernel with a temperature.  Its row0 argument (the first batch row
  // of the launch) is 0: every launch starts at row 0.
  auto launch_pw = [&](auto kernel, auto... extra) {
    return launch_pdl(kernel, dim3(cdiv((long)nrows * d.D, 256)), dim3(256), (size_t)0, st, (const float*)a->gtmp,
                      (const float*)a->ptab, tok, tok_stride, (const float*)(o1 + d.A + d.C), (int64_t)d.O1,
                      (const float*)(a->call + cur * d.D), a->gates + cur * d.G, a->call + nxt * d.D, a->hall + nxt * d.D,
                      bv.on ? bv.hall + nxt * d.D : (bf16*)nullptr, hd_t, hd_stride, dmask_t, nrows, d.D, d.V,
                      (const unsigned long long*)((hd_t && a->has_dropout == 2) ? a->dropout_state : nullptr), a->dropout_p, 0, t, ss,
                      extra...);
  };
  if (sampling && a->ss_temp) {
    const GumbelStep gs{a->ss_temp, a->ss_gu ? a->ss_gu + (int64_t)t * d.V : nullptr, (int64_t)d.T * d.V};
    LO_CUDA(launch_pw(lstm_pw_fwd_gumbel_kernel, gs));
  } else {
    LO_CUDA(launch_pw(sampling ? lstm_pw_fwd_kernel<true> : lstm_pw_fwd_kernel<false>));
  }
  LO_LAUNCH_OK();
  if (sampling) {
    // the head of step t, right after the cell (the next step's cell reads these logits, see lstm_pw_fwd_kernel): the returned
    // predictions of this mode
    LO_TRY(head_nt(a, bv.on, hd_t, ss.hd_bf, hd_stride, a->logits + (int64_t)t * d.Vl, (int64_t)d.T * d.Vl, nrows, st));
  }
  return LO_OK;
}

// one backward step t for the first nrows rows, the launches of forward_step in reverse; dal, dal_b, dal_t: the d alpha rows of
// lo_decoder_backward
static int backward_step(const lo_decoder_args* a, const Dims& d, int t, int nrows, const float* dal, int64_t dal_b, int64_t dal_t,
                         cudaStream_t st) {
  const int dt = a->dt;
  const BfViews bv = bf_views(a, d);
  const int64_t cur = (int64_t)t * d.B, nxt = (int64_t)(t + 1) * d.B;
  float* dcat_t = a->dcat + cur * d.O1;
  bf16* dcat_bf_t = bv.on ? bv.dcat + cur * d.O1 : nullptr;
  const float* o1 = a->out1 + cur * d.O1;
  float* dxh = a->dxh;
  const float* dmul = (a->has_dropout == 1 && a->dropout_mask) ? a->dropout_mask + (int64_t)t * d.D : nullptr;
  if (!(g_opt_dbg_skip & 4))   // row0 = 0 as in forward_step
    LO_CUDA(launch_pdl(lstm_pw_bwd_kernel, dim3(cdiv((long)nrows * d.D, 256)), dim3(256), (size_t)0, st,
                       (const float*)(a->dhd + (int64_t)t * d.D), (int64_t)d.T * d.D, dmul, (const float*)(dxh + d.C),
                       (int64_t)(d.C + d.D), a->dc, (const float*)(a->gates + cur * d.G), (const float*)(a->call + cur * d.D),
                       (const float*)(a->call + nxt * d.D), dcat_t + d.A + d.C, (int64_t)d.O1,
                       bv.on ? dcat_bf_t + d.A + d.C : (bf16*)nullptr, bv.on ? dxh : (float*)nullptr, d.C, nrows, d.D,
                       (const unsigned long long*)(a->has_dropout == 2 ? a->dropout_state : nullptr), a->dropout_p, 0, t));
  LO_LAUNCH_OK();
  // [dgctx | dh_prev] = dG @ [W_ih[:, E:] | W_hh]
  if (!(g_opt_dbg_skip & 4))
    LO_TRY(step_gemm_nt(bv.on, dcat_t + d.A + d.C, bv.on ? dcat_bf_t + d.A + d.C : nullptr, d.O1, a->wbwd1, dt, d.G, dxh, d.C + d.D,
                        nrows, d.C + d.D, d.G, nullptr, 0, 4, 1, st));
  const float* alpha_t = a->alphas + t * d.R;
  const float* ctx_t = a->ctx + cur * d.C;
  const float* dal_t_ptr = dal + (int64_t)t * dal_t;
  const float* sreg_t = a->sreg + t;
  float* de_t = a->de + t * d.R;
  float* dctx_t = a->dctx + cur * d.C;
  if (g_opt_dbg_skip & 2) {
  } else if (g_opt_att_pipe) {
    AttBwdArgs x{a->att1, a->enc, o1, o1 + d.A, d.O1, a->w_full, alpha_t, (int64_t)d.T * d.R, ctx_t, dxh, d.C + d.D, dal_t_ptr, dal_b,
                 sreg_t, d.T, de_t, dcat_t, dcat_t + d.A, d.O1, dcat_bf_t, dcat_bf_t ? dcat_bf_t + d.A : nullptr, dctx_t, nrows, d.R,
                 a->work, a->dmean, 0, 0, att_mask_at(a, t)};
    x.ordered_dwf = g_opt_det;
    LO_TRY(attention_bwd_pipe(x, dt, d.C, st));
  } else {
    const int ns = att_splits(d.B);
    int* cnt_c = (int*)a->work;
    float* part_c = (float*)((char*)a->work + att_partials_offset(nrows));
    dim3 grid(ns, nrows);
#define LO_ATT_BWD(TY_, NV)                                                                                                       \
  attention_bwd_kernel<TY_, NV><<<grid, LO_ATT_THREADS, 0, st>>>(                                                                 \
      (const TY_*)a->att1, (const TY_*)a->enc, o1, o1 + d.A, d.O1, a->w_full, alpha_t, (int64_t)d.T * d.R, ctx_t, dxh, d.C + d.D,    \
      dal_t_ptr, dal_b, sreg_t, d.T, de_t, dcat_t, dcat_t + d.A, d.O1, dcat_bf_t, dcat_bf_t ? dcat_bf_t + d.A : nullptr, dctx_t, d.R, \
      ns, cnt_c, part_c)
    if (dt == LO_F32) {
      if (d.C == 256) LO_ATT_BWD(float, 1); else if (d.C == 512) LO_ATT_BWD(float, 2); else LO_ATT_BWD(float, 4);
    } else {
      if (d.C == 256) LO_ATT_BWD(bf16, 1); else if (d.C == 512) LO_ATT_BWD(bf16, 2); else LO_ATT_BWD(bf16, 4);
    }
#undef LO_ATT_BWD
    LO_LAUNCH_OK();
  }
  // dh_prev += [datt2 | dgate_pre] @ [W_d ; W_beta]
  if (!(g_opt_dbg_skip & 4))
    LO_TRY(step_gemm_nt(bv.on, dcat_t, dcat_bf_t, d.O1, a->wbwd2, dt, d.A + d.C, dxh + d.C, d.C + d.D, nrows, d.D, d.A + d.C, nullptr, 1,
                        4, 1, st));
  return LO_OK;
}

// one beam-search step of either decoder flavour (beam_step_kernel, one CTA per image): the top-k over beam x V log-probs in shared
// memory, twice that with the diversity penalty (div_on)
static int beam_select(const float* logits, int V, int beam, int n_img, int t, int max_steps, int64_t end_id, float* logp,
                       int32_t* finished, int64_t* ids, int64_t* parents, int32_t* fin_hist, int64_t* next_tok, int32_t* parent_rows,
                       bool div_on, float div_gamma, float div_prob, const float* div_u_t, const uint64_t* div_state, cudaStream_t st) {
  static bool smem_attr = false;      // the 200 kB opt-in, once per process
  const size_t smem = (size_t)beam * V * 4 * (div_on ? 2 : 1);
  if (!smem_attr && smem > 48 * 1024) {
    LO_CUDA(cudaFuncSetAttribute(beam_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    smem_attr = true;
  }
  beam_step_kernel<<<n_img, 256, smem, st>>>(logits, V, beam, t, end_id, logp, finished, ids, parents, fin_hist, next_tok, parent_rows,
                                             max_steps, div_on ? logf(div_gamma) : 0.f, div_on ? div_prob : 0.f, div_u_t,
                                             (const unsigned long long*)div_state);
  LO_LAUNCH_OK();
  return LO_OK;
}

// the hypotheses of a finished beam search (lo_beam_backtrack): one CTA per (image, slot).  The image's parents [n][beam] go to shared
// memory with coalesced loads and thread 0 walks them there (a walk over global memory is n dependent loads), leaving per step the slot
// whose token the hypothesis holds and the row that emitted it; then the CTA writes the ids and copies the n attention rows, 16 bytes at
// a time when VEC (R % 4 == 0 and every row 16-byte aligned), zeros past the image's region count.  A parent outside [0, beam) reads as
// slot 0, so foreign data cannot send the walk out of bounds.
template <bool VEC>
__global__ void __launch_bounds__(256) beam_backtrack_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ parents,
                                                             int64_t ids_stride_steps, int beam, int n, const float* __restrict__ alphas,
                                                             int64_t alpha_row_stride, int R, const int32_t* __restrict__ reg_off,
                                                             int lineage, int64_t* __restrict__ ids_out, float* __restrict__ att_out) {
  extern __shared__ int32_t s_bt[];           // parents [n][beam], then slot [n] and row [n]
  int32_t* s_slot = s_bt + n * beam;
  int32_t* s_row = s_slot + n;
  const int img = blockIdx.x / beam, s = blockIdx.x % beam, tid = threadIdx.x;
  const int64_t src0 = (int64_t)img * ids_stride_steps * beam;
  if (lineage) {
    for (int j = tid; j < n * beam; j += blockDim.x) {
      const int64_t p = parents[src0 + j];
      s_bt[j] = (p >= 0 && p < beam) ? (int32_t)p : 0;
    }
    __syncthreads();
    if (tid == 0) {
      int cur = s;
      for (int t = n - 1; t >= 0; t--) {
        s_slot[t] = cur;
        cur = s_bt[t * beam + cur];
        s_row[t] = cur;
      }
    }
  } else {
    for (int t = tid; t < n; t += blockDim.x) s_slot[t] = s_row[t] = s;
  }
  __syncthreads();
  const int64_t hyp = (int64_t)img * beam + s;
  for (int t = tid; t < n; t += blockDim.x) ids_out[hyp * n + t] = ids[src0 + (int64_t)t * beam + s_slot[t]];
  if (!att_out) return;
  const int Ri = reg_off ? reg_off[img + 1] - reg_off[img] : R;
  const float* src = alphas + (int64_t)img * beam * alpha_row_stride;
  float* dst = att_out + hyp * n * R;
  if (VEC) {
    const int R4 = R / 4;
    for (int j = tid; j < n * R4; j += blockDim.x) {
      const int t = j / R4, q = j - t * R4;
      const float* a = src + s_row[t] * alpha_row_stride + (int64_t)t * R + 4 * q;
      float4 v;
      if (4 * q + 3 < Ri) {
        v = *(const float4*)a;
      } else {
        v.x = 4 * q < Ri ? a[0] : 0.f;
        v.y = 4 * q + 1 < Ri ? a[1] : 0.f;
        v.z = 4 * q + 2 < Ri ? a[2] : 0.f;
        v.w = 0.f;
      }
      *(float4*)(dst + (int64_t)t * R + 4 * q) = v;
    }
  } else {
    for (int j = tid; j < n * R; j += blockDim.x) {
      const int t = j / R, r = j - t * R;
      dst[j] = r < Ri ? src[s_row[t] * alpha_row_stride + (int64_t)t * R + r] : 0.f;
    }
  }
}

// ------------------------------------------------------------------------------------------------ decode loops of both flavours
// A flavour F hands the loops F::c: the step's logits [B][V], device scratch of B rows each and the ragged attention state
// (rg.reg_off NULL: every image has R regions) of rpi rows per image; F::prologue(st); F::step(t, st): the cell step fed next_tok
// (or the start token), then the head into logits; and for beam search F::reorder(t, st): the state of step t gathered by parent_rows.
struct DecodeCtx {
  int B, T, V, rpi;
  const float* logits;
  int64_t* next_tok;
  int32_t *finished, *parent_rows;
  AttRagged rg;
  const AttRagged* ragged() const { return rg.reg_off ? &rg : nullptr; }
};

struct BeamArgs {
  int beam;
  float div_gamma, div_prob;
  const float* div_u;            // [max_steps][B][V] injected uniforms, or NULL (Philox from div_state)
  const uint64_t* div_state;
  bool div_on() const { return !(div_gamma == 1.f || div_prob == 0.f); }        // beam_search_decoder_cell.py:270-273
};

// the decode arguments both flavours check alike (bm NULL: greedy decode), before anything is enqueued; then everything before
// step 0: finished = 0, log-probs = 0 (beam search, :106-107), the prologue, the ragged CTA map
template <class F>
static int decode_begin(F& f, int max_steps, bool outputs, const BeamArgs* bm, float* logp, cudaStream_t st) {
  DecodeCtx& c = f.c;
  LO_CHECK_ARG(outputs && max_steps > 0 && max_steps <= c.T, "outputs / max_steps (<= T capacity)");
  if (bm) {
    LO_CHECK_ARG(!bm->div_on() || (bm->div_gamma > 0.f && (bm->div_u || bm->div_state)),
                 "diversity penalty needs gamma > 0 and div_u or div_state");
    LO_CHECK_ARG(bm->beam >= 1 && bm->beam <= LO_BEAM_MAX && c.B % bm->beam == 0, "1 <= beam (rows_per_img) <= 16, B % beam == 0");
    LO_CHECK_ARG((size_t)bm->beam * c.V * 4 * (bm->div_on() ? 2 : 1) <= 200 * 1024, "beam*V too large for the shared-memory top-k");
  }
  LO_CUDA(cudaMemsetAsync(c.finished, 0, (size_t)c.B * 4, st));
  if (logp) LO_CUDA(cudaMemsetAsync(logp, 0, (size_t)c.B * 4, st));
  LO_TRY(f.prologue(st));
  if (c.rg.reg_off) LO_TRY(attention_ragged_prepare(c.rg, c.B, c.rpi, st));
  return LO_OK;
}

template <class F>
static int greedy_loop(F& f, int64_t end_id, int max_steps, int64_t* tokens, int32_t* fin_hist, cudaStream_t st) {
  const DecodeCtx& c = f.c;
  LO_TRY(decode_begin(f, max_steps, tokens && c.finished, nullptr, nullptr, st));
  for (int t = 0; t < max_steps; t++) {
    LO_TRY(f.step(t, st));
    argmax_kernel<<<cdiv(c.B, 8), 256, 0, st>>>(c.logits, c.V, tokens + t, max_steps, c.next_tok, c.finished, end_id, c.B);
    LO_LAUNCH_OK();
    if (fin_hist) {
      fin_hist_kernel<<<cdiv(c.B, 128), 128, 0, st>>>(c.finished, fin_hist + t, max_steps, c.B);
      LO_LAUNCH_OK();
    }
  }
  return LO_OK;
}

// bm.beam == c.rpi once decode_begin has checked it
template <class F>
static int beam_loop(F& f, const BeamArgs& bm, int64_t end_id, int max_steps, int64_t* ids, int64_t* parents, int32_t* fin_hist,
                     float* logp, cudaStream_t st) {
  const DecodeCtx& c = f.c;
  LO_TRY(decode_begin(f, max_steps, ids && parents && fin_hist && logp, &bm, logp, st));
  for (int t = 0; t < max_steps; t++) {
    LO_TRY(f.step(t, st));
    LO_TRY(beam_select(c.logits, c.V, bm.beam, c.B / bm.beam, t, max_steps, end_id, logp, c.finished, ids, parents, fin_hist,
                       c.next_tok, c.parent_rows, bm.div_on(), bm.div_gamma, bm.div_prob,
                       bm.div_u ? bm.div_u + (int64_t)t * c.B * c.V : nullptr, bm.div_state, st));
    LO_TRY(f.reorder(t, st));
  }
  return LO_OK;
}

// the torch flavour in the decode loops: next tokens (int64 [B], start_id before step 0) in sreg ([B][>= 2] floats); greedy
// decode's `finished` comes from the caller, beam search keeps finished and the parent rows (int32 [B] each) in row_loss
struct TorchDecode {
  const lo_decoder_args* a;
  int64_t start_id;
  Dims d;
  BfViews bv;
  DecodeCtx c;
  TorchDecode(const lo_decoder_args* a_, int64_t start, int32_t* finished, int32_t* parent_rows)
      : a(a_), start_id(start), d(dims(a_)), bv(bf_views(a_, d)),
        c{d.B, d.T, d.V, a_->rows_per_img > 1 ? a_->rows_per_img : 1, a_->logits, (int64_t*)a_->sreg, finished, parent_rows,
          ragged_of(a_)} {}
  int prologue(cudaStream_t st) {
    fill_i64_kernel<<<cdiv(d.B, 128), 128, 0, st>>>(c.next_tok, start_id, d.B);
    LO_LAUNCH_OK();
    return forward_prologue(a, d, st);
  }
  // the cell step, then logits_t = fc(h_t)   (no dropout at decode time)
  int step(int t, cudaStream_t st) {
    LO_TRY(forward_step(a, d, t, d.B, c.ragged(), c.next_tok, 1, nullptr, 0, nullptr, st));
    const int64_t h_t = (int64_t)(t + 1) * d.B * d.D;
    return head_nt(a, bv.on, a->hall + h_t, bv.on ? bv.hall + h_t : nullptr, d.D, a->logits, d.V, d.B, st);
  }
  // h and c of step t by parents (through gtmp as a temporary), then the bf16 copy of h
  int reorder(int t, cudaStream_t st) {
    const int64_t n = (int64_t)d.B * d.D;
    float* h_new = a->hall + (t + 1) * n;
    float* c_new = a->call + (t + 1) * n;
    gather_rows_kernel<<<cdiv((long)n, 256), 256, 0, st>>>(h_new, c.parent_rows, a->gtmp, nullptr, d.B, d.D);
    LO_LAUNCH_OK();
    gather_rows_kernel<<<cdiv((long)n, 256), 256, 0, st>>>(c_new, c.parent_rows, a->gtmp + n, nullptr, d.B, d.D);
    LO_LAUNCH_OK();
    LO_CUDA(cudaMemcpyAsync(h_new, a->gtmp, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    LO_CUDA(cudaMemcpyAsync(c_new, a->gtmp + n, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    if (bv.on) LO_TRY(lo_cast(h_new, LO_F32, bv.hall + (t + 1) * n, LO_BF16, n, st));
    return LO_OK;
  }
};

}  // namespace lo

using namespace lo;

extern "C" {

int64_t lo_decoder_bfwork_bytes(const lo_decoder_args* a) {
  if (!a) return 0;
  const int64_t TB = (int64_t)a->T * a->B, O1 = a->A + a->C + 4 * a->D;
  const int64_t Vp = (a->V + 7) / 8 * 8;
  const int64_t Vl = a->ldl > 0 ? a->ldl : a->V;
  return (TB * (O1 + a->D + a->C + Vp + a->D + Vl) + (int64_t)a->B * a->D + (int64_t)a->A * a->C + (int64_t)a->D * Vl +
          TB * ((a->R + 7) / 8 * 8) + TB * a->C + (int64_t)(a->V + a->E) * 4 * a->D) * 2 + 1024;
}

int64_t lo_sizeof_decoder_args(void) { return (int64_t)sizeof(lo_decoder_args); }

int64_t lo_attention_workspace_bytes(int B, int C) {
  return att_partials_offset(B) + (int64_t)B * LO_ATT_MAXSPLIT * (C + 2) * 4;
}
/* the decoder entry points use two such regions: the first for the attention launches of the time loop, the second for the CTA map
   of a decode call with per-image region counts (ragged_of) */
int64_t lo_decoder_workspace_bytes(int B, int C) { return 2 * lo_attention_workspace_bytes(B, C); }

int lo_attention_forward(const void* att1, const void* enc, int dt, const float* att2, int64_t att2_stride, const float* wf,
                         float* alpha, int64_t alpha_stride, float* ctx, float* gate_pre, int64_t gate_stride, float* gctx,
                         int B, int R, int A, int C, void* work, void* stream) {
  LO_CHECK_ARG(att1 && enc && att2 && wf && alpha && ctx && work, "null pointer");
  LO_CHECK_ARG(A == C && (C == 256 || C == 512 || C == 1024), "attention_dim == encoder_dim in {256,512,1024}");
  LO_CHECK_ARG(B > 0 && B <= 512 && R > 0, "B in 1..512, R > 0");
  LO_CHECK_ARG(att2_stride % 4 == 0, "att2 rows must be 16-byte aligned");
  return attention_forward_launch(att1, enc, dt, att2, att2_stride, wf, alpha, alpha_stride, ctx, gate_pre, gate_stride, gctx, nullptr,
                                  B, R, C, work, (cudaStream_t)stream, 1, nullptr, 1);
}

int lo_attention_forward_mask(const void* att1, const void* enc, int dt, const float* att2, int64_t att2_stride, const float* wf,
                              float* alpha, int64_t alpha_stride, float* ctx, float* gate_pre, int64_t gate_stride, float* gctx,
                              uint8_t* relu_mask_out, int B, int R, int A, int C, void* work, void* stream) {
  LO_CHECK_ARG(att1 && enc && att2 && wf && alpha && ctx && work, "null pointer");
  LO_CHECK_ARG(A == C && (C == 256 || C == 512 || C == 1024), "attention_dim == encoder_dim in {256,512,1024}");
  LO_CHECK_ARG(B > 0 && B <= 512 && R > 0, "B in 1..512, R > 0");
  LO_CHECK_ARG(att2_stride % 4 == 0, "att2 rows must be 16-byte aligned");
  LO_CHECK_ARG(!relu_mask_out || g_opt_att_pipe, "mask bits are written by the TMA-ring kernel (option att_pipe=1)");
  return attention_forward_launch(att1, enc, dt, att2, att2_stride, wf, alpha, alpha_stride, ctx, gate_pre, gate_stride, gctx, nullptr,
                                  B, R, C, work, (cudaStream_t)stream, 1, relu_mask_out, 1);
}

int lo_attention_backward(const void* att1, const void* enc, int dt, const float* att2, const float* gate, int64_t o1_stride,
                          const float* wf, const float* alpha, int64_t alpha_stride, const float* ctx, const float* dgctx,
                          int64_t dg_stride, const float* dreg, int64_t dreg_stride, const float* sreg, int64_t sreg_stride, float* de,
                          float* datt2, float* dgp, int64_t dcat_stride, float* dctx_out, float* dwf_part, const uint8_t* relu_mask,
                          int B, int R, int A, int C, void* work, void* stream) {
  LO_CHECK_ARG(att1 && enc && att2 && wf && alpha && ctx && dgctx && de && datt2 && work, "null pointer");
  LO_CHECK_ARG(A == C && (C == 256 || C == 512 || C == 1024), "attention_dim == encoder_dim in {256,512,1024}");
  LO_CHECK_ARG(B > 0 && B <= 512 && R > 0, "B in 1..512, R > 0");
  LO_CHECK_ARG(g_opt_att_pipe, "stand-alone attention backward runs on the TMA-ring kernel (option att_pipe=1)");
  AttBwdArgs x{att1, enc, att2, gate, o1_stride, wf, alpha, alpha_stride, ctx, dgctx, dg_stride, dreg, dreg_stride, sreg, sreg_stride,
               de, datt2, dgp, dcat_stride, nullptr, nullptr, dctx_out, B, R, work, dwf_part, 0, 0, relu_mask};
  x.abi = 1;
  return attention_bwd_pipe(x, dt, C, (cudaStream_t)stream);
}

// work of lo_attention_step_backward: attention split workspace | d w_full partials [B][A] | de [B][R] | datt2 [B][A] | sreg [B] |
// d att1 [B][R][A] (dt) | W_enc^T [C][A] bf16, each region 256-byte aligned
static inline int64_t step_ws_align(int64_t n) { return (n + 255) & ~(int64_t)255; }

int64_t lo_attention_step_workspace_bytes(int B, int R, int A, int C, int dt) {
  if (B < 1 || R < 1 || A < 1 || C < 1) return 0;
  const int64_t es = dt == LO_F32 ? 4 : 2;
  return step_ws_align(lo_attention_workspace_bytes(B, C)) + 2 * step_ws_align((int64_t)B * A * 4) + step_ws_align((int64_t)B * R * 4) +
         step_ws_align((int64_t)B * 4) + step_ws_align((int64_t)B * R * A * es) + step_ws_align((int64_t)A * C * 2);
}

int lo_attention_step_backward(const void* enc, const void* att1, int dt, const float* h, const float* att2, const void* w_enc,
                               const void* w_dec, const float* wf, const float* alpha, const float* ctx, const float* dctx,
                               const float* dalpha, float* denc, float* dh, float* g_w_enc, float* g_b_enc, float* g_w_dec, float* g_b_dec,
                               float* g_w_full, float* g_b_full, float* de, float* datt2, void* datt1, int B, int R, int A, int C, int D,
                               int impl, void* work, void* stream) {
  LO_CHECK_ARG(enc && att1 && h && att2 && w_enc && w_dec && wf && alpha && ctx && dctx && work, "null pointer");
  LO_CHECK_ARG(dt == LO_F32 || dt == LO_BF16, "dt must be LO_F32 or LO_BF16");
  LO_CHECK_ARG(impl == LO_IMPL_SIMT || impl == LO_IMPL_TC, "impl must be LO_IMPL_SIMT or LO_IMPL_TC");
  LO_CHECK_ARG(A == C && (C == 256 || C == 512 || C == 1024), "attention_dim == encoder_dim in {256,512,1024}");
  LO_CHECK_ARG(B > 0 && B <= 512 && R > 0 && D > 0, "B in 1..512, R > 0, D > 0");
  LO_CHECK_ARG((((uintptr_t)enc | (uintptr_t)att1 | (uintptr_t)datt1) & 15) == 0,
               "enc, att1 and datt1 must be 16-byte aligned (bulk copies, 16-byte stores)");
  LO_CHECK_ARG(g_opt_att_pipe, "stand-alone attention backward runs on the TMA-ring kernel (option att_pipe=1)");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t es = dt == LO_F32 ? 4 : 2;
  const int64_t BR = (int64_t)B * R;
  char* w = (char*)work + step_ws_align(lo_attention_workspace_bytes(B, C));
  float* ws_dwf = (float*)w;     w += step_ws_align((int64_t)B * A * 4);
  float* ws_de = (float*)w;      w += step_ws_align(BR * 4);
  float* ws_datt2 = (float*)w;   w += step_ws_align((int64_t)B * A * 4);
  float* ws_sreg = (float*)w;    w += step_ws_align((int64_t)B * 4);
  void* ws_datt1 = w;            w += step_ws_align(BR * A * es);
  bf16* ws_wet = (bf16*)w;
  float* de_ = de ? de : ws_de;
  float* datt2_ = datt2 ? datt2 : ws_datt2;
  // d att1 is written only when something reads it: d enc, the encoder_att gradients, or the caller
  const bool need_d1 = denc || g_w_enc || g_b_enc || datt1;
  void* d1 = datt1 ? datt1 : ws_datt1;
  const bool tc = impl == LO_IMPL_TC && dt == LO_BF16 && tc_available();
  // s = <dctx, ctx> + sum_r alpha_r dalpha_r: the second term per batch row (one warp each, fixed order)
  if (dalpha) {
    sreg_kernel<<<cdiv(B, 8), 256, 0, st>>>(alpha, dalpha, R, 0, ws_sreg, B, 1, R);
    LO_LAUNCH_OK();
  }
  if (g_w_full) LO_CUDA(cudaMemsetAsync(ws_dwf, 0, (size_t)B * A * 4, st));
  AttBwdArgs x{att1, enc, att2, nullptr, A, wf, alpha, R, ctx, dctx, C, dalpha, R, dalpha ? ws_sreg : nullptr, 1, de_, datt2_, nullptr, A,
               nullptr, nullptr, nullptr, B, R, work, g_w_full ? ws_dwf : nullptr, 0, 0, nullptr};
  x.abi = 1;
  x.datt1 = need_d1 ? d1 : nullptr;
  x.ordered_dwf = g_opt_det;
  LO_TRY(attention_bwd_pipe(x, dt, C, st));
  // full_att: d weight = sum_b of the per-row partials; d bias = 0 exactly (sum_r de_r = 0), as lo_decoder_backward
  if (g_w_full) LO_TRY(colsum(ws_dwf, LO_F32, g_w_full, B, A, A, 0, st));
  if (g_b_full) LO_CUDA(cudaMemsetAsync(g_b_full, 0, 4, st));
  // decoder_att: dh = datt2 W_d ; d W_d = datt2^T h ; d b_d = colsum(datt2)
  if (dh) LO_TRY(gemm_nn(datt2_, LO_F32, A, w_dec, dt, D, dh, LO_F32, D, B, D, A, 0, LO_IMPL_SIMT, st));
  if (g_w_dec) LO_TRY(gemm_tn(datt2_, LO_F32, A, h, LO_F32, D, g_w_dec, LO_F32, D, A, D, B, 0, LO_IMPL_SIMT, st));
  if (g_b_dec) LO_TRY(colsum(datt2_, LO_F32, g_b_dec, B, A, A, 0, st));
  // encoder_att: d W_e = datt1^T enc ; d b_e = colsum(datt1) ; denc = datt1 W_e + alpha (x) dctx
  if (g_w_enc) {
    if (tc) {
      LO_CUDA(cudaMemsetAsync(g_w_enc, 0, (size_t)A * C * 4, st));
      LO_TRY(tc_gemm_tn((const bf16*)d1, A, (const bf16*)enc, C, g_w_enc, C, A, C, (int)BR, st));
    } else {
      LO_TRY(gemm_tn(d1, dt, A, enc, dt, C, g_w_enc, LO_F32, C, A, C, (int)BR, 0, LO_IMPL_SIMT, st));
    }
  }
  if (g_b_enc) LO_TRY(colsum(d1, dt, g_b_enc, (int)BR, A, A, 0, st));
  if (denc) {
    if (tc) {
      transpose_kernel<bf16><<<dim3(cdiv(C, 32), cdiv(A, 32)), dim3(32, 8), 0, st>>>((const bf16*)w_enc, C, ws_wet, A, A, C);
      LO_LAUNCH_OK();
      LO_TRY(tc_gemm_nt((const bf16*)d1, A, ws_wet, A, denc, LO_F32, C, (int)BR, C, A, nullptr, 0, 0, st));
    } else {
      LO_TRY(gemm_nn(d1, dt, A, w_enc, dt, C, denc, LO_F32, C, (int)BR, C, A, 0, LO_IMPL_SIMT, st));
    }
    add_outer_kernel<<<LO_NUM_SMS * 8, 256, 0, st>>>(denc, alpha, dctx, R, C, BR * C);
    LO_LAUNCH_OK();
  }
  return LO_OK;
}

int lo_decoder_forward(const lo_decoder_args* a, int with_loss, void* stream) {
  LO_TRY(check_args(a));
  LO_TRY(check_reg_off(a, false));
  cudaStream_t st = (cudaStream_t)stream;
  const Dims d = dims(a);
  const bool ragged = a->bt_host[d.T - 1] < d.B;
  const bool sampling = a->ss_prob != nullptr;
  if (ragged && a->phase != 2) {
    LO_CUDA(cudaMemsetAsync(a->alphas, 0, (size_t)d.B * d.T * d.R * 4, st));
    LO_CUDA(cudaMemsetAsync(a->hd, 0, (size_t)d.B * d.T * d.D * 4, st));
    const BfViews bz = bf_views(a, d);
    if (sampling && bz.on) LO_CUDA(cudaMemsetAsync(bz.hd, 0, (size_t)d.B * d.T * d.D * 2, st));   // written by the cell in this mode
  }
  if (sampling)     // the steps overwrite the positions they decode; the others keep the teacher token
    LO_CUDA(cudaMemcpy2DAsync(a->fed, (size_t)d.T * 8, a->caps, (size_t)a->caps_stride * 8, (size_t)d.T * 8, d.B,
                              cudaMemcpyDeviceToDevice, st));
  LO_TRY(upload_dlen(a, st));
  if (a->phase != 2) {
  LO_TRY(forward_prologue(a, d, st));
  // the time loop (DESIGN.md §4): per-step launches over the rows still decoding
  for (int t = 0; t < d.T; t++) {
    const float* dm = (a->has_dropout == 1 && a->dropout_mask) ? a->dropout_mask + (int64_t)t * d.D : nullptr;
    LO_TRY(forward_step(a, d, t, a->bt_host[t], nullptr, a->caps + t, a->caps_stride, a->hd + (int64_t)t * d.D, (int64_t)d.T * d.D, dm,
                        st));
  }
  }   // phase != 2
  if (a->phase == 1) return LO_OK;       // extension: the caller runs a second layer over hd before the head
  if (g_opt_dbg_skip & 8) return LO_OK;
  // predictions = fc(dropout(h))  (seq2seq_torch.py:316), hoisted out of the loop
  const BfViews bvf = bf_views(a, d);
  const bool fc_tc = bvf.on && d.Vl % 64 == 0 && d.D % 64 == 0;
  if (sampling) {
    // the time loop wrote the logits (and, in bf16, the hd mirror the fc weight gradient reads)
  } else if (fc_tc) {
    LO_TRY(lo_cast(a->hd, LO_F32, bvf.hd, LO_BF16, (int64_t)d.B * d.T * d.D, stream));
    LO_TRY(tc_gemm_nt_ex(bvf.hd, d.D, (const bf16*)a->w_fc, d.D, a->logits, LO_F32, d.Vl, d.B * d.T, d.V, d.D, a->b_fc, 0, 0, 1, 0, 0, st));
  } else {
    LO_TRY(gemm_nt(a->hd, LO_F32, d.D, a->w_fc, a->dt, d.D, a->logits, LO_F32, d.Vl, d.B * d.T, d.V, d.D, a->b_fc, 0, 0, LO_IMPL_SIMT, st));
  }
  // rows that stopped decoding keep zeros in `predictions` (seq2seq_torch.py:301): what the GEMM wrote there (bias) is ignored by
  // the CE kernel and handled by the Python side for the returned tensor
  if (with_loss) {
    long nvalid = 0;
    for (int t = 0; t < d.T; t++) nvalid += a->bt_host[t];
    const float inv_n = 1.0f / (float)nvalid;
    ce_kernel<<<cdiv((long)d.B * d.T, 8), 256, 0, st>>>(a->logits, a->caps, a->caps_stride, work_dlen(a), a->row_loss, a->dlogits,
                                                         (fc_tc && a->dlogits) ? bvf.dlogits : nullptr, d.B, d.T, d.V, d.Vl, inv_n);
    LO_LAUNCH_OK();
    reg_kernel<<<cdiv((long)d.B * d.R, 256), 256, 0, st>>>(a->alphas, a->row_loss + (int64_t)d.B * d.T, a->dreg, d.B, d.T, d.R, a->alpha_c);
    LO_LAUNCH_OK();
    loss_finalize_kernel<<<1, 1024, 0, st>>>(a->row_loss, d.B * d.T, a->row_loss + (int64_t)d.B * d.T, d.B * d.R, inv_n, a->alpha_c, a->loss);
    LO_LAUNCH_OK();
  }
  return LO_OK;
}

int lo_decoder_pack_bwd_weights(const lo_decoder_args* a, void* stream) {
  LO_TRY(check_args(a));
  LO_CHECK_ARG(a->wbwd1 && a->wbwd2, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const Dims d = dims(a);
  const size_t es = a->dt == LO_F32 ? 4 : 2;
  dim3 blk(32, 8);
  // wbwd1 [C+D][4D]: rows 0..C-1 <- (w_ih[:, E:])^T ; rows C.. <- w_hh^T
  const char* w_hh = (const char*)a->wcat1 + (size_t)(d.A + d.C) * d.D * es;
  const char* w_dec = (const char*)a->wcat1;
  const char* w_beta = (const char*)a->wcat1 + (size_t)d.A * d.D * es;
  LO_DISPATCH_DT(a->dt, T, {
    transpose_kernel<T><<<dim3(cdiv(d.C, 32), cdiv(d.G, 32)), blk, 0, st>>>((const T*)a->w_ih + d.E, d.E + d.C, (T*)a->wbwd1, d.G, d.G, d.C);
    transpose_kernel<T><<<dim3(cdiv(d.D, 32), cdiv(d.G, 32)), blk, 0, st>>>((const T*)w_hh, d.D, (T*)a->wbwd1 + (int64_t)d.C * d.G, d.G, d.G, d.D);
    // wbwd2 [D][A+C]: [n][k<A] = w_dec[k][n] ; [n][A+k] = w_beta[k][n]
    transpose_kernel<T><<<dim3(cdiv(d.D, 32), cdiv(d.A, 32)), blk, 0, st>>>((const T*)w_dec, d.D, (T*)a->wbwd2, d.A + d.C, d.A, d.D);
    transpose_kernel<T><<<dim3(cdiv(d.D, 32), cdiv(d.C, 32)), blk, 0, st>>>((const T*)w_beta, d.D, (T*)a->wbwd2 + d.A, d.A + d.C, d.C, d.D);
  });
  lo::g_launches += 3;
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_decoder_backward(const lo_decoder_args* a, void* stream) {
  LO_TRY(check_args(a));
  LO_TRY(check_reg_off(a, false));
  LO_CHECK_ARG(!a->dpred_ext || a->dlogits, "dpred_ext needs dlogits");
  LO_CHECK_ARG(!a->dpred_ext || a->dpred_stride >= a->V, "dpred_stride >= V");
  LO_CHECK_ARG(a->phase != 2 || !a->dalpha_ext, "phase 2 reads no d alpha: pass dalpha_ext to the phase-1 call");
  cudaStream_t st = (cudaStream_t)stream;
  const Dims d = dims(a);
  const int dt = a->dt;
  const bool ragged = a->bt_host[d.T - 1] < d.B;
  const int64_t BT = (int64_t)d.B * d.T;
  // d alpha rows: the regulariser's (one row per b), the caller's (one per (b, t)), or none (generic mode without dalpha_ext)
  const bool generic = a->dpred_ext != nullptr;
  const float* dal = a->dalpha_ext ? a->dalpha_ext : (generic ? nullptr : a->dreg);
  const int64_t dal_b = a->dalpha_ext ? (int64_t)d.T * d.R : (dal ? d.R : 0), dal_t = a->dalpha_ext ? d.R : 0;
  const BfViews bvf = bf_views(a, d);
  const bool fc_tc = bvf.on && d.Vl % 64 == 0 && d.D % 64 == 0;
  if (generic && a->phase != 1) {
    // plain launch (no overlap with the preceding one); everything after it that reads dlogits waits for it
    dpred_kernel<<<dim3(cdiv(d.Vl, 128), (unsigned)(BT < 65535 ? BT : 65535)), 128, 0, st>>>(
        a->dpred_ext, a->dpred_stride, work_dlen(a), a->dlogits, fc_tc ? bvf.dlogits : nullptr, d.T, d.V, d.Vl, BT, 0);
    LO_LAUNCH_OK();
  }
  if (a->phase != 2) {
    LO_TRY(lo_decoder_pack_bwd_weights(a, stream));
    // sreg[b,t] = sum_r alpha dreg
    if (dal) {
      sreg_kernel<<<cdiv(BT, 8), 256, 0, st>>>(a->alphas, dal, dal_b, dal_t, a->sreg, d.B, d.T, d.R);
      LO_LAUNCH_OK();
    } else {
      LO_CUDA(cudaMemsetAsync(a->sreg, 0, (size_t)BT * 4, st));
    }
  }
  // fc backward (hoisted): g_w_fc = dlogits^T hd ; g_b_fc ; dhd = dlogits @ W_fc (* dropout mask)
  if (a->phase == 1) {
    // extension: d hd was put there by the caller (backward of the layer between the cell and fc)
  } else if (fc_tc) {
    // (the dlogits bf16 mirror was written by ce_kernel or, in the generic mode, by dpred_kernel)
    LO_CUDA(cudaMemsetAsync(a->g_w_fc, 0, (size_t)d.V * d.D * 4, st));
    LO_TRY(tc_gemm_tn(bvf.dlogits, d.Vl, bvf.hd, d.D, a->g_w_fc, d.D, d.V, d.D, (int)BT, st));
    transpose_kernel<bf16><<<dim3(cdiv(d.D, 32), cdiv(d.V, 32)), dim3(32, 8), 0, st>>>((const bf16*)a->w_fc, d.D, bvf.wfct, d.Vl, d.V, d.D);
    LO_LAUNCH_OK();
    LO_TRY(tc_gemm_nt_ex(bvf.dlogits, d.Vl, bvf.wfct, d.Vl, a->dhd, LO_F32, d.D, (int)BT, d.D, d.Vl, nullptr, 0, 0, 1, 0, 0, st));
  } else {
    LO_TRY(gemm_tn(a->dlogits, LO_F32, d.Vl, a->hd, LO_F32, d.D, a->g_w_fc, LO_F32, d.D, d.V, d.D, (int)BT, 0, LO_IMPL_SIMT, st));
    LO_TRY(gemm_nn(a->dlogits, LO_F32, d.Vl, a->w_fc, dt, d.D, a->dhd, LO_F32, d.D, (int)BT, d.D, d.V, 0, LO_IMPL_SIMT, st));
  }
  if (a->phase != 1) LO_TRY(colsum(a->dlogits, LO_F32, a->g_b_fc, (int)BT, d.V, d.Vl, 0, st));
  if (a->phase == 2) return LO_OK;
  LO_CUDA(cudaMemsetAsync(a->dxh, 0, (size_t)d.B * (d.C + d.D) * 4, st));
  LO_CUDA(cudaMemsetAsync(a->dc, 0, (size_t)d.B * d.D * 4, st));
  if (ragged) {
    LO_CUDA(cudaMemsetAsync(a->dcat, 0, (size_t)d.T * d.B * d.O1 * 4, st));
    LO_CUDA(cudaMemsetAsync(a->de, 0, (size_t)BT * d.R * 4, st));
    LO_CUDA(cudaMemsetAsync(a->dctx, 0, (size_t)d.T * d.B * d.C * 4, st));
    const BfViews bz = bf_views(a, d);
    if (bz.on) LO_CUDA(cudaMemsetAsync(bz.dcat, 0, (size_t)d.T * d.B * d.O1 * 2, st));
  }
  const BfViews bv = bf_views(a, d);
  if (g_opt_att_pipe) LO_CUDA(cudaMemsetAsync(a->dmean, 0, (size_t)d.B * d.A * 4, st));    // [B][A] scratch for d w_full
  for (int t = d.T - 1; t >= 0; t--) LO_TRY(backward_step(a, d, t, a->bt_host[t], dal, dal_b, dal_t, st));
  // dinit = [dh0 | dc0]
  LO_CUDA(cudaMemcpy2DAsync(a->dinit, (size_t)2 * d.D * 4, a->dxh + d.C, (size_t)(d.C + d.D) * 4, (size_t)d.D * 4, d.B,
                            cudaMemcpyDeviceToDevice, st));
  LO_CUDA(cudaMemcpy2DAsync(a->dinit + d.D, (size_t)2 * d.D * 4, a->dc, (size_t)d.D * 4, (size_t)d.D * 4, d.B,
                            cudaMemcpyDeviceToDevice, st));
  if (g_opt_dbg_skip & 1) return LO_OK;
  // ---- hoisted gradients
  const bool tc = bv.on;
  bf16* dcat_bf = bv.dcat;
  bf16* hall_bf = bv.hall;
  bf16* gctx_bf = bv.gctx;
  bf16* wet_bf = bv.wet;
  // [W_d; W_beta; W_hh] and biases: dcat^T @ h_prev
  if (tc) {
    LO_CUDA(cudaMemsetAsync(a->g_wcat1, 0, (size_t)d.O1 * d.D * 4, st));
    LO_TRY(tc_gemm_tn(dcat_bf, d.O1, hall_bf, d.D, a->g_wcat1, d.D, d.O1, d.D, d.T * d.B, st));
  } else {
    LO_TRY(gemm_tn(a->dcat, LO_F32, d.O1, a->hall, LO_F32, d.D, a->g_wcat1, LO_F32, d.D, d.O1, d.D, d.T * d.B, 0, LO_IMPL_SIMT, st));
  }
  LO_TRY(colsum(a->dcat, LO_F32, a->g_bcat1, d.T * d.B, d.O1, d.O1, 0, st));
  // W_ih[:, E:] : dG^T @ gctx ; b_ih = colsum(dG) (== g_b_hh)
  if (tc) {
    LO_CUDA(cudaMemset2DAsync(a->g_w_ih + d.E, (size_t)(d.E + d.C) * 4, 0, (size_t)d.C * 4, d.G, st));
    LO_TRY(tc_gemm_tn(dcat_bf + d.A + d.C, d.O1, gctx_bf, d.C, a->g_w_ih + d.E, d.E + d.C, d.G, d.C, d.T * d.B, st));
  } else {
    LO_TRY(gemm_tn(a->dcat + d.A + d.C, LO_F32, d.O1, a->gctx, LO_F32, d.C, a->g_w_ih + d.E, LO_F32, d.E + d.C, d.G, d.C, d.T * d.B, 0,
                   LO_IMPL_SIMT, st));
  }
  LO_TRY(colsum(a->dcat + d.A + d.C, LO_F32, a->g_b_ih, d.T * d.B, d.G, d.O1, 0, st));
  // embedding path through the projection table, scattered by the tokens the forward fed (scheduled sampling: fed, else caps)
  const int64_t* in_tok = a->ss_prob ? a->fed : a->caps;
  const int64_t in_stride = a->ss_prob ? (int64_t)d.T : a->caps_stride;
  if (tc) {
    const int Vp = (d.V + 7) / 8 * 8;
    onehot_kernel<<<LO_NUM_SMS * 8, 256, 0, st>>>(in_tok, in_stride, work_dlen(a), bv.onehot, d.B, d.T, Vp);
    LO_LAUNCH_OK();
    LO_CUDA(cudaMemsetAsync(a->dptab, 0, (size_t)d.V * d.G * 4, st));
    LO_TRY(tc_gemm_tn(bv.onehot, Vp, dcat_bf + d.A + d.C, d.O1, a->dptab, d.G, d.V, d.G, d.T * d.B, st));
  } else {
    dim3 grid(cdiv(d.G, 256), d.V);
    dptab_kernel<<<grid, 256, 0, st>>>(a->dcat, d.O1, (int64_t)d.B * d.O1, d.A + d.C, in_tok, in_stride, work_dlen(a), a->dptab,
                                       d.B, d.T, d.G);
    LO_LAUNCH_OK();
  }
  if (tc && d.E % 64 == 0 && d.G % 64 == 0 && d.V >= 64) {
    // g_emb = dptab W_ih[:, :E] and g_W_ih[:, :E] = dptab^T emb on wgmma (bf16 copy of dptab, transposed weight slice)
    LO_TRY(lo_cast(a->dptab, LO_F32, bv.dptab, LO_BF16, (int64_t)d.V * d.G, stream));
    transpose_kernel<bf16><<<dim3(cdiv(d.E, 32), cdiv(d.G, 32)), dim3(32, 8), 0, st>>>((const bf16*)a->w_ih, d.E + d.C, bv.wihT, d.G, d.G, d.E);
    LO_LAUNCH_OK();
    LO_TRY(tc_gemm_nt(bv.dptab, d.G, bv.wihT, d.G, a->g_emb, LO_F32, d.E, d.V, d.E, d.G, nullptr, 0, 0, st));
    LO_CUDA(cudaMemset2DAsync(a->g_w_ih, (size_t)(d.E + d.C) * 4, 0, (size_t)d.E * 4, d.G, st));
    LO_TRY(tc_gemm_tn(bv.dptab, d.G, (const bf16*)a->emb, d.E, a->g_w_ih, d.E + d.C, d.G, d.E, d.V, st));
  } else {
    LO_TRY(gemm_nn(a->dptab, LO_F32, d.G, a->w_ih, dt, d.E + d.C, a->g_emb, LO_F32, d.E, d.V, d.E, d.G, 0, LO_IMPL_SIMT, st));
    LO_TRY(gemm_tn(a->dptab, LO_F32, d.G, a->emb, dt, d.E, a->g_w_ih, LO_F32, d.E + d.C, d.G, d.E, d.V, 0, LO_IMPL_SIMT, st));
  }
  // d att1 + d w_full in one sweep over att1
  LO_CUDA(cudaMemsetAsync(a->g_b_full, 0, 4, st));   // sum_r de = 0 exactly (softmax); reference value is rounding noise
  const bool pipe_dwf = g_opt_att_pipe && !att_mask_at(a, 0);   // d w_full accumulated per batch row by the attention backward
  if (!g_opt_det) {
    dim3 grid(d.A / 64, cdiv(d.R, 32), d.B);
    if (g_opt_att_pipe) {
      // the per-step kernels' part of d w_full (all of it without mask bits, the att2 term with them) sits in dmean ([B][A] scratch)
      LO_TRY(colsum(a->dmean, LO_F32, a->g_w_full, d.B, d.A, d.A, 0, st));
    } else {
      LO_CUDA(cudaMemsetAsync(a->g_w_full, 0, (size_t)d.A * 4, st));
    }
    if (pipe_dwf) {
      LO_DISPATCH_DT(dt, T, (datt1_kernel<T, 0><<<grid, 128, 0, st>>>((const T*)a->att1, a->out1, d.O1, (int64_t)d.B * d.O1, a->de,
                                                                       a->w_full, (T*)a->datt1, nullptr, d.T, d.R, d.A, 1, 0)));
    } else if (g_opt_att_pipe) {
      // mask-bit scheme: the sweep adds the x term
      LO_DISPATCH_DT(dt, T, (datt1_kernel<T, 2><<<grid, 128, 0, st>>>((const T*)a->att1, a->out1, d.O1, (int64_t)d.B * d.O1, a->de,
                                                                       a->w_full, (T*)a->datt1, a->g_w_full, d.T, d.R, d.A, 1, 0)));
    } else {
      LO_DISPATCH_DT(dt, T, (datt1_kernel<T, 1><<<grid, 128, 0, st>>>((const T*)a->att1, a->out1, d.O1, (int64_t)d.B * d.O1, a->de,
                                                                       a->w_full, (T*)a->datt1, a->g_w_full, d.T, d.R, d.A, 1, 0)));
    }
    LO_LAUNCH_OK();
  } else {
    // ordered: the sweep adds its d w_full part per batch row onto the dmean rows, then one colsum over b
    const int nch = cdiv(cdiv(d.R, 32), 16);            // row chunks per block: <= 16 row blocks (one cluster) per batch row
    static bool attr = false;
    if (!attr) {
      LO_CUDA(cudaFuncSetAttribute(datt1_kernel<float, 1>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
      LO_CUDA(cudaFuncSetAttribute(datt1_kernel<bf16, 1>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
      LO_CUDA(cudaFuncSetAttribute(datt1_kernel<float, 2>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
      LO_CUDA(cudaFuncSetAttribute(datt1_kernel<bf16, 2>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
      attr = true;
    }
    dim3 grid(d.A / 64, cdiv(d.R, 32 * nch), d.B);
    const dim3 cl(1, grid.y, 1);
    if (pipe_dwf) {
      LO_DISPATCH_DT(dt, T, (datt1_kernel<T, 0><<<grid, 128, 0, st>>>((const T*)a->att1, a->out1, d.O1, (int64_t)d.B * d.O1, a->de,
                                                                       a->w_full, (T*)a->datt1, nullptr, d.T, d.R, d.A, nch, 0)));
    } else if (g_opt_att_pipe) {
      LO_DISPATCH_DT(dt, T, LO_CUDA(launch_cluster(datt1_kernel<T, 2>, grid, dim3(128), 0, st, cl, false, (const T*)a->att1,
                                                   (const float*)a->out1, (int64_t)d.O1, (int64_t)d.B * d.O1, (const float*)a->de,
                                                   (const float*)a->w_full, (T*)a->datt1, a->dmean, d.T, d.R, d.A, nch, 1)));
    } else {
      LO_CUDA(cudaMemsetAsync(a->dmean, 0, (size_t)d.B * d.A * 4, st));
      LO_DISPATCH_DT(dt, T, LO_CUDA(launch_cluster(datt1_kernel<T, 1>, grid, dim3(128), 0, st, cl, false, (const T*)a->att1,
                                                   (const float*)a->out1, (int64_t)d.O1, (int64_t)d.B * d.O1, (const float*)a->de,
                                                   (const float*)a->w_full, (T*)a->datt1, a->dmean, d.T, d.R, d.A, nch, 1)));
    }
    LO_LAUNCH_OK();
    LO_TRY(colsum(a->dmean, LO_F32, a->g_w_full, d.B, d.A, d.A, 0, st));
  }
  // encoder_att: g_W = datt1^T enc ; g_b = colsum(datt1) ; denc = datt1 @ W_e
  if (tc) {
    LO_CUDA(cudaMemsetAsync(a->g_w_enc_att, 0, (size_t)d.A * d.C * 4, st));
    LO_TRY(tc_gemm_tn((const bf16*)a->datt1, d.A, (const bf16*)a->enc, d.C, a->g_w_enc_att, d.C, d.A, d.C, d.B * d.R, st));
    transpose_kernel<bf16><<<dim3(cdiv(d.C, 32), cdiv(d.A, 32)), dim3(32, 8), 0, st>>>((const bf16*)a->w_enc_att, d.C, wet_bf, d.A, d.A, d.C);
    LO_LAUNCH_OK();
    LO_TRY(tc_gemm_nt((const bf16*)a->datt1, d.A, wet_bf, d.A, a->denc, LO_F32, d.C, d.B * d.R, d.C, d.A, nullptr, 0, 0, st));
  } else {
    LO_TRY(gemm_tn(a->datt1, dt, d.A, a->enc, dt, d.C, a->g_w_enc_att, LO_F32, d.C, d.A, d.C, d.B * d.R, 0, LO_IMPL_SIMT, st));
    LO_TRY(gemm_nn(a->datt1, dt, d.A, a->w_enc_att, dt, d.C, a->denc, LO_F32, d.C, d.B * d.R, d.C, d.A, 0, LO_IMPL_SIMT, st));
  }
  LO_TRY(colsum(a->datt1, dt, a->g_b_enc_att, d.B * d.R, d.A, d.A, 0, st));
  // denc[b] += alphas[b]^T @ dctx[:, b, :]   (the context read, summed over time — a batched GEMM instead of a per-step RMW)
  if (tc && d.C % 8 == 0) {
    // wgmma, one launch (3-D tensor maps, grid.y = batch); bf16 operands cast once after the loop
    const int Rp = (int)rpad8(d.R);
    cast_pad_rows_kernel<<<LO_NUM_SMS * 8, 256, 0, st>>>(a->alphas, bv.alphas, BT, d.R, Rp);
    LO_LAUNCH_OK();
    cast_tb_to_bt_kernel<<<LO_NUM_SMS * 8, 256, 0, st>>>(a->dctx, bv.dctx, d.T, d.B, d.C);
    LO_LAUNCH_OK();
    LO_TRY(tc_gemm_tn_batched(bv.alphas, Rp, (int64_t)d.T * Rp, bv.dctx, d.C, (int64_t)d.T * d.C, a->denc, d.C, (int64_t)d.R * d.C, d.R,
                              d.C, d.T, d.B, st));
  } else {
    GemmDesc g{d.R, d.C, d.T, 1, d.R, (int64_t)d.B * d.C, 1, d.C, d.B, (int64_t)d.T * d.R, d.C, (int64_t)d.R * d.C, nullptr, 1, 0};
    LO_TRY(gemm(a->alphas, LO_F32, a->dctx, LO_F32, a->denc, LO_F32, g, LO_IMPL_SIMT, st));
  }
  // init_h / init_c
  LO_TRY(gemm_tn(a->dinit, LO_F32, 2 * d.D, a->mean, LO_F32, d.C, a->g_w_init, LO_F32, d.C, 2 * d.D, d.C, d.B, 0, LO_IMPL_SIMT, st));
  LO_TRY(colsum(a->dinit, LO_F32, a->g_b_init, d.B, 2 * d.D, 2 * d.D, 0, st));
  LO_TRY(gemm_nn(a->dinit, LO_F32, 2 * d.D, a->w_init, dt, d.C, a->dmean, LO_F32, d.C, d.B, d.C, 2 * d.D, 0, LO_IMPL_SIMT, st));
  {
    const int64_t total = (int64_t)d.B * d.R * d.C;
    add_rowbcast_kernel<<<LO_NUM_SMS * 8, 256, 0, st>>>(a->denc, a->dmean, d.R, d.C, 1.0f / (float)d.R, total);
    LO_LAUNCH_OK();
  }
  if (a->has_dropout == 2 || (a->ss_prob && a->dropout_state)) {
    // forward and backward of this step drew the same Philox stream (dropout, sampling coins); the next step (also a graph
    // replay) gets a new one
    bump_counter_kernel<<<1, 1, 0, st>>>((unsigned long long*)a->dropout_state + 1);
    LO_LAUNCH_OK();
  }
  return LO_OK;
}

int lo_decoder_greedy_hist(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps, int64_t* tokens,
                           int32_t* finished, int32_t* fin_hist, void* stream) {
  LO_TRY(check_args(a));
  LO_TRY(check_reg_off(a, true));
  LO_CHECK_ARG(!a->ss_prob, "scheduled sampling (ss_prob) is a training mode: greedy decode feeds its own argmax already");
  TorchDecode f(a, start_id, finished, nullptr);
  return greedy_loop(f, end_id, max_steps, tokens, fin_hist, (cudaStream_t)stream);
}

int lo_decoder_greedy(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps, int64_t* tokens,
                      int32_t* finished, void* stream) {
  return lo_decoder_greedy_hist(a, start_id, end_id, max_steps, tokens, finished, nullptr, stream);
}

int lo_decoder_beam(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps, int64_t* ids, int64_t* parents,
                    int32_t* fin_hist, float* logp, void* stream) {
  return lo_decoder_beam_div(a, start_id, end_id, max_steps, ids, parents, fin_hist, logp, 1.f, 0.f, nullptr, nullptr, stream);
}

int lo_decoder_beam_div(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps, int64_t* ids, int64_t* parents,
                        int32_t* fin_hist, float* logp, float div_gamma, float div_prob, const float* div_u,
                        const uint64_t* div_state, void* stream) {
  LO_TRY(check_args(a));
  LO_TRY(check_reg_off(a, true));
  LO_CHECK_ARG(!a->ss_prob, "scheduled sampling (ss_prob) is a training mode: not available in beam search");
  LO_CHECK_ARG((int64_t)a->B * a->T >= 2 * a->B, "row_loss scratch too small");
  int32_t* finished = (int32_t*)a->row_loss;
  TorchDecode f(a, start_id, finished, finished + a->B);
  return beam_loop(f, BeamArgs{a->rows_per_img, div_gamma, div_prob, div_u, div_state}, end_id, max_steps, ids, parents, fin_hist, logp,
                   (cudaStream_t)stream);
}

int lo_beam_backtrack(const int64_t* ids, const int64_t* parents, int64_t ids_stride_steps, int n_img, int beam, int n,
                      const float* alphas, int64_t alpha_row_stride, int R, const int32_t* reg_off, const int32_t* reg_off_host,
                      int mode, int64_t* ids_out, float* att_out, void* stream) {
  LO_CHECK_ARG(ids && parents && ids_out, "null ids / parents / ids_out");
  LO_CHECK_ARG(!alphas == !att_out, "alphas and att_out must be set together");
  LO_CHECK_ARG(n_img >= 1 && beam >= 1 && beam <= LO_BEAM_MAX, "n_img >= 1 and 1 <= beam <= 16");
  LO_CHECK_ARG(n >= 1 && n <= ids_stride_steps, "1 <= n <= ids_stride_steps");
  LO_CHECK_ARG(mode == LO_BEAM_SLOTS || mode == LO_BEAM_LINEAGE, "mode must be LO_BEAM_SLOTS or LO_BEAM_LINEAGE");
  const size_t smem = (size_t)n * (beam + 2) * 4;
  LO_CHECK_ARG(smem <= 48 * 1024, "n * (beam + 2) * 4 bytes of parents and walk exceed 48 kB of shared memory");
  bool vec = false;
  if (att_out) {
    LO_CHECK_ARG(R >= 1 && (int64_t)n * R <= INT32_MAX, "1 <= R and n * R < 2^31");
    LO_CHECK_ARG(alpha_row_stride >= (int64_t)n * R, "alpha_row_stride >= n * R");
    LO_CHECK_ARG(!reg_off == !reg_off_host, "reg_off and reg_off_host must be set together");
    if (reg_off_host)
      for (int i = 0; i < n_img; i++) {
        const int c = reg_off_host[i + 1] - reg_off_host[i];
        LO_CHECK_ARG(c >= 1 && c <= R, "region count of every image in 1..R (reg_off_host)");
      }
    vec = R % 4 == 0 && alpha_row_stride % 4 == 0 && (uintptr_t)alphas % 16 == 0 && (uintptr_t)att_out % 16 == 0;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int lineage = mode == LO_BEAM_LINEAGE;
  if (vec)
    beam_backtrack_kernel<true><<<n_img * beam, 256, smem, st>>>(ids, parents, ids_stride_steps, beam, n, alphas, alpha_row_stride, R,
                                                                 reg_off, lineage, ids_out, att_out);
  else
    beam_backtrack_kernel<false><<<n_img * beam, 256, smem, st>>>(ids, parents, ids_stride_steps, beam, n, alphas, alpha_row_stride, R,
                                                                  reg_off, lineage, ids_out, att_out);
  LO_LAUNCH_OK();
  return LO_OK;
}

}  // extern "C"

// TensorFlow-flavour (Genthial) decoder: same translation unit, shares the kernels above
#include "lo_tfdecoder.cuh"
// generic sequence LSTM (extension: row-encoder biLSTM, second decoder layer)
#include "lo_lstmseq.cuh"
