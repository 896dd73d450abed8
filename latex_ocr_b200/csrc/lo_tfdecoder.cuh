// TensorFlow-flavour decoder (SURVEY.md §8-a row a7): the Genthial attention cell, teacher-forced training pass with a
// hand-derived backward, masked cross-entropy, greedy and beam decode.  Part of the lo_decoder.cu translation unit (it
// reuses that file's kernels: attention launchers, datt1 sweep, transposes, beam step, argmax ..., and its decode loops).
//
// Reference semantics (paths relative to the reference root):
//   model/components/attention_cell.py:58-89   step:  x = [emb ; o] ; (c,h) = LSTMCell(x,(c,h)) ; hd = dropout(h) ; ctx = attention(hd) ;
//                                              o = dropout(tanh(hd o_W_h + ctx o_W_c)) ; logits = o y_W_o ; next state (c, h, o):
//                                              the recurrent h is the UNDROPPED one (:71, :87), the recurrent o the dropped one
//   model/components/attention_mechanism.py:43 att_img = img W_img (once) ; :79-94 e = beta . tanh(att_img + h W_h), softmax
//   :145-153 / attention_cell.py:51-56         c0, h0, o0 = tanh(mean_r(img) W + b)
//   model/decoder.py:48-57, 75-96              training inputs [start_token ; E[formula[:, :-1]]], dynamic_rnn over all T columns
//   model/img2seq.py:68-71                     loss = mean over sequence_mask(length) of the sparse softmax CE
//   tf.contrib.rnn.LSTMCell (TF 1.12)          gate order i, j, f, o ; forget_bias 1.0 ; one kernel over [x ; h]
//
// Schedule (same ideas as the torch flavour, DESIGN.md §4): att_img hoisted; the embedding half of the LSTM kernel folded into a
// [V+1][4D] table (row V = start token); logits and every weight gradient hoisted out of the time loop into stacked GEMMs;
// d att_img by one post-loop sweep; d enc by a batched alpha^T dctx GEMM.  Sampling (lo_tfdec_args.ss_prob: scheduled sampling,
// self-critical training): the logits GEMM moves into the loop and the cell kernel chooses the token consumed (ss_block_tokens).  The TMA-ring attention kernels serve both flavours:
// the (NVA, NVC) = (1, 2) instantiation streams dim_e = 256 att_img columns next to C = 512 image channels, ACT = tanh.

namespace lo {

// ------------------------------------------------------------------------------------------------ pointwise kernels
// MODE 0: the token is tok (NULL: the start token).  MODE 1 / 2 (sampling, lo_tfdec_args.ss_prob): tok is the teacher token
// formula[b][t_idx] and the token fed is chosen from the logits of step t_idx and recorded (ss_block_tokens: argmax, or a
// Gumbel-max draw).  Those logits come from the head GEMM two launches back (head GEMM(t_idx), z GEMM(t_idx + 1), this kernel), so
// they are read after griddepcontrol.wait: the wait returns once the z GEMM has completed, and the z GEMM's own wait (it reads
// xh[t_idx + 1], written before the head GEMM) returned only once the head GEMM had.
template <int MODE>
__device__ __forceinline__ void tf_lstm_pw_fwd_body(const float* __restrict__ z, const float* __restrict__ ptab,
                                                    const int64_t* __restrict__ tok, int64_t tok_stride, int V,
                                                    const float* __restrict__ c_prev, float* __restrict__ gates, float* __restrict__ c_out,
                                                    float* __restrict__ h_out, bf16* __restrict__ h_bf, int64_t xh_stride,
                                                    const float* __restrict__ keep, float* __restrict__ hd_out, bf16* __restrict__ hd_bf,
                                                    int nrows, int D, int t_idx, const SsStep& ss, const GumbelStep& gs) {
  pdl_wait();
  pdl_trigger();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int64_t tk_ss = 0;
  if constexpr (MODE != 0) {
    const bool live = idx < nrows * D;
    ss_block_tokens<MODE>(tok, tok_stride, nrows, D, V, 0, t_idx, ss, gs, live, live ? idx / D : 0, tk_ss);
  }
  if (idx >= nrows * D) return;
  const int b = idx / D, j = idx % D;
  int64_t tk = V;                                       // row V of the table = start token (decoder.py:45-46, :90-93)
  if constexpr (MODE != 0) {
    tk = tk_ss;
    if (tk < 0) tk = 0;
    if (tk >= V) tk = V - 1;
  } else if (tok) {
    tk = tok[(int64_t)b * tok_stride];
    if (tk < 0) tk = 0;
    if (tk >= V) tk = V - 1;
  }
  const float* pt = ptab + tk * 4 * D;
  const float* z0 = z + (int64_t)b * 4 * D;
  const float i = sigmoidf_(z0[j] + pt[j]);
  const float g = tanhf(z0[D + j] + pt[D + j]);
  const float f = sigmoidf_(z0[2 * D + j] + pt[2 * D + j] + 1.0f);       // forget_bias = 1.0
  const float o = sigmoidf_(z0[3 * D + j] + pt[3 * D + j]);
  const float c = f * c_prev[(int64_t)b * D + j] + i * g;
  const float h = o * tanhf(c);
  float* gt = gates + (int64_t)b * 4 * D;
  gt[j] = i; gt[D + j] = g; gt[2 * D + j] = f; gt[3 * D + j] = o;
  c_out[(int64_t)b * D + j] = c;
  // attention_cell.py:71-72,87: new_cell_state keeps the UNDROPPED h as the recurrent state; tf.nn.dropout(new_h) feeds only
  // the attention and the o projection of this step -> separate buffer hd (only when dropout is on)
  h_out[(int64_t)b * xh_stride + j] = h;
  if (h_bf) h_bf[(int64_t)b * xh_stride + j] = __float2bfloat16_rn(h);
  if (keep) {
    const float hdv = h * keep[(int64_t)b * D + j];
    hd_out[(int64_t)b * D + j] = hdv;
    if (hd_bf) hd_bf[(int64_t)b * D + j] = __float2bfloat16_rn(hdv);
  }
}

__global__ void tf_lstm_pw_fwd_kernel(const float* __restrict__ z, const float* __restrict__ ptab, const int64_t* __restrict__ tok,
                                      int64_t tok_stride, int V, const float* __restrict__ c_prev, float* __restrict__ gates,
                                      float* __restrict__ c_out, float* __restrict__ h_out, bf16* __restrict__ h_bf, int64_t xh_stride,
                                      const float* __restrict__ keep, float* __restrict__ hd_out, bf16* __restrict__ hd_bf, int nrows,
                                      int D) {
  tf_lstm_pw_fwd_body<0>(z, ptab, tok, tok_stride, V, c_prev, gates, c_out, h_out, h_bf, xh_stride, keep, hd_out, hd_bf, nrows, D, 0,
                         SsStep{}, GumbelStep{});
}
// sampling (lo_tfdec_args.ss_prob): MODE 1 feeds the argmax, MODE 2 (ss_temp) a draw from softmax(logits / tau)
template <int MODE>
__global__ void tf_lstm_pw_fwd_ss_kernel(const float* __restrict__ z, const float* __restrict__ ptab, const int64_t* __restrict__ tok,
                                         int64_t tok_stride, int V, const float* __restrict__ c_prev, float* __restrict__ gates,
                                         float* __restrict__ c_out, float* __restrict__ h_out, bf16* __restrict__ h_bf,
                                         int64_t xh_stride, const float* __restrict__ keep, float* __restrict__ hd_out,
                                         bf16* __restrict__ hd_bf, int nrows, int D, int t_idx, SsStep ss, GumbelStep gs) {
  tf_lstm_pw_fwd_body<MODE>(z, ptab, tok, tok_stride, V, c_prev, gates, c_out, h_out, h_bf, xh_stride, keep, hd_out, hd_bf, nrows, D,
                            t_idx, ss, gs);
}

// sampling: the choice of the last step, fed[b][T-1] from the logits of step T-1 (recorded, never consumed: the last token of a
// self-critical sample).  The same block geometry as the pointwise kernels, no cell.
template <int MODE>
__global__ void tf_ss_last_token_kernel(const int64_t* __restrict__ tok, int64_t tok_stride, int V, int nrows, int D, int t_idx,
                                        SsStep ss, GumbelStep gs) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = idx < nrows * D;
  int64_t tk = 0;
  ss_block_tokens<MODE>(tok, tok_stride, nrows, D, V, 0, t_idx, ss, gs, live, live ? idx / D : 0, tk);
}

__global__ void tf_o_pw_fwd_kernel(const float* __restrict__ oc, const float* __restrict__ oh, int64_t oh_stride,
                                   const float* __restrict__ keep, float* __restrict__ o_out, bf16* __restrict__ o_bf,
                                   int64_t xh_stride, int nrows, int O) {
  pdl_wait();
  pdl_trigger();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nrows * O) return;
  const int b = idx / O, j = idx % O;
  float o = tanhf(oc[(int64_t)b * O + j] + oh[(int64_t)b * oh_stride + j]);
  if (keep) o *= keep[(int64_t)b * O + j];
  o_out[(int64_t)b * xh_stride + j] = o;
  if (o_bf) o_bf[(int64_t)b * xh_stride + j] = __float2bfloat16_rn(o);
}

// d o_t = (gradient through the next step's LSTM input) + d logits_t y_W_o^T ; d pre = d o (1 - o^2)
__global__ void tf_o_pw_bwd_kernel(float* __restrict__ dxh, int64_t xh_stride, const float* __restrict__ dologit,
                                   const float* __restrict__ keep, const float* __restrict__ o_st, float* __restrict__ dpre,
                                   bf16* __restrict__ dpre_bf, int64_t dp_stride, int nrows, int O) {
  pdl_wait();
  pdl_trigger();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nrows * O) return;
  const int b = idx / O, j = idx % O;
  float dv = dxh[(int64_t)b * xh_stride + j] + dologit[(int64_t)b * O + j];
  dxh[(int64_t)b * xh_stride + j] = 0.f;                // the GEMM that refills dxh accumulates (split-K atomics)
  float o = o_st[(int64_t)b * xh_stride + j];
  if (keep) {
    const float k = keep[(int64_t)b * O + j];
    dv *= k;
    o = k != 0.f ? o / k : 0.f;
  }
  const float d = dv * (1.f - o * o);
  dpre[(int64_t)b * dp_stride + j] = d;
  if (dpre_bf) dpre_bf[(int64_t)b * dp_stride + j] = __float2bfloat16_rn(d);
}

__global__ void tf_lstm_pw_bwd_kernel(float* __restrict__ dxh, int64_t xh_stride, int O, const float* __restrict__ dhc,
                                      int64_t dhc_stride, const float* __restrict__ keep, float* __restrict__ dc,
                                      const float* __restrict__ gates, const float* __restrict__ c_prev,
                                      const float* __restrict__ c_cur, float* __restrict__ dz, bf16* __restrict__ dz_bf, int nrows,
                                      int D) {
  pdl_wait();
  pdl_trigger();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nrows * D) return;
  const int b = idx / D, j = idx % D;
  // d h_t = (recurrent path: next step's LSTM read the undropped h) + keep * (attention / o-projection paths, which read
  // the dropped h of this step)
  float dhd = dhc[(int64_t)b * dhc_stride + j];
  if (keep) dhd *= keep[(int64_t)b * D + j];
  const float dh = dxh[(int64_t)b * xh_stride + O + j] + dhd;
  dxh[(int64_t)b * xh_stride + O + j] = 0.f;
  const float* gt = gates + (int64_t)b * 4 * D;
  const float i = gt[j], g = gt[D + j], f = gt[2 * D + j], o = gt[3 * D + j];
  const float tc = tanhf(c_cur[(int64_t)b * D + j]);
  const float dct = dc[(int64_t)b * D + j] + dh * o * (1.f - tc * tc);
  float v[4];
  v[0] = dct * g * i * (1.f - i);
  v[1] = dct * i * (1.f - g * g);
  v[2] = dct * c_prev[(int64_t)b * D + j] * f * (1.f - f);
  v[3] = dh * tc * o * (1.f - o);
  dc[(int64_t)b * D + j] = dct * f;
#pragma unroll
  for (int q = 0; q < 4; q++) {
    dz[(int64_t)b * 4 * D + q * D + j] = v[q];
    if (dz_bf) dz_bf[(int64_t)b * 4 * D + q * D + j] = __float2bfloat16_rn(v[q]);
  }
}

// c0 | h0 | o0 = tanh(pre)  ->  call[0], xh[0] = [o0 | h0]
__global__ void tf_init_state_kernel(const float* __restrict__ pre, float* __restrict__ sinit, float* __restrict__ c0,
                                     float* __restrict__ xh0, bf16* __restrict__ xh0_bf, int64_t xh_stride, int B, int D, int O) {
  const int W = 2 * D + O;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * W) return;
  const int b = idx / W, col = idx % W;
  const float s = tanhf(pre[idx]);
  sinit[idx] = s;
  if (col < D) { c0[(int64_t)b * D + col] = s; return; }
  const int x = col < 2 * D ? O + (col - D) : col - 2 * D;
  xh0[(int64_t)b * xh_stride + x] = s;
  if (xh0_bf) xh0_bf[(int64_t)b * xh_stride + x] = __float2bfloat16_rn(s);
}
__global__ void tf_init_bwd_kernel(const float* __restrict__ dc, const float* __restrict__ dxh, int64_t xh_stride,
                                   const float* __restrict__ sinit, float* __restrict__ dinit, int B, int D, int O) {
  const int W = 2 * D + O;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * W) return;
  const int b = idx / W, col = idx % W;
  const float g = col < D ? dc[(int64_t)b * D + col]
                          : dxh[(int64_t)b * xh_stride + (col < 2 * D ? O + (col - D) : col - 2 * D)];
  const float s = sinit[idx];
  dinit[idx] = g * (1.f - s * s);
}

// masked CE forward + backward, warp per (t,b) row of the time-major logits (img2seq.py:68-71)
__global__ void tf_ce_kernel(const float* __restrict__ logits, const int64_t* __restrict__ formula, int64_t f_stride,
                             const int32_t* __restrict__ lengths, float* __restrict__ row_loss, float* __restrict__ dlogits,
                             bf16* __restrict__ dlogits_bf, int B, int Tn, int V, int ld, float inv_n) {
  const int row = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= B * Tn) return;
  const int t = row / B, b = row % B;
  const float* lg = logits + (int64_t)row * ld;
  float* dl = dlogits + (int64_t)row * ld;
  bf16* dlb = dlogits_bf ? dlogits_bf + (int64_t)row * ld : nullptr;
  if (t >= lengths[b]) {
    if (lane == 0) row_loss[row] = 0.f;
    for (int v = lane; v < ld; v += 32) {
      dl[v] = 0.f;
      if (dlb) dlb[v] = __float2bfloat16_rn(0.f);
    }
    return;
  }
  float mx = -INFINITY;
  for (int v = lane; v < V; v += 32) mx = fmaxf(mx, lg[v]);
  mx = warp_max(mx);
  float se = 0.f;
  for (int v = lane; v < V; v += 32) se += expf(lg[v] - mx);
  se = warp_sum(se);
  const float lse = mx + logf(se);
  int64_t tg = formula[(int64_t)b * f_stride + t];
  if (tg < 0) tg = 0;
  if (tg >= V) tg = V - 1;
  if (lane == 0) row_loss[row] = lse - lg[tg];
  for (int v = lane; v < ld; v += 32) {
    const float g = v < V ? (expf(lg[v] - lse) - (v == (int)tg ? 1.f : 0.f)) * inv_n : 0.f;
    dl[v] = g;
    if (dlb) dlb[v] = __float2bfloat16_rn(g);
  }
}

// d ptab[token consumed at (t,b)][:] += dz[t][b][:]   (token = start row V at t = 0, else formula[b][t-1])
__global__ void tf_dptab_scatter_kernel(const float* __restrict__ dz, const int64_t* __restrict__ formula, int64_t f_stride,
                                        float* __restrict__ dptab, int B, int Tn, int G, int V) {
  const int64_t total = (int64_t)B * Tn * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int col = (int)(i % G);
    const int64_t row = i / G;
    const int t = (int)(row / B), b = (int)(row % B);
    int64_t tk = V;
    if (t > 0) {
      tk = formula[(int64_t)b * f_stride + t - 1];
      if (tk < 0) tk = 0;
      if (tk >= V) tk = V - 1;
    }
    atomicAdd(dptab + tk * G + col, dz[i]);
  }
}

// The same sum under option deterministic: d ptab[v][:] = sum of dz[t][b][:] over the (t, b) that consumed token v, added in
// ascending (t, b) order, so the sum does not depend on scheduling.  One block per (table row, TF_DPT_COLS columns): 256 threads
// scan the tokens of steps 1.. in time-major order with one ballot per 256 of them and add the dz rows of the hits.  It writes every
// element.  Not the default: at the tools/tf_bench.py shape the train step took 24.2 ms with it against 23.8 ms with the scatter
// (H100 80GB HBM3, 700 W power limit).
#define TF_DPT_COLS 1024
__global__ void __launch_bounds__(256) tf_dptab_kernel(const float* __restrict__ dz, const int64_t* __restrict__ formula,
                                                       int64_t f_stride, float* __restrict__ dptab, int B, int Tn, int G, int V) {
  constexpr int NC = TF_DPT_COLS / 256;
  const int v = blockIdx.y;
  const int j0 = blockIdx.x * TF_DPT_COLS + threadIdx.x;
  __shared__ unsigned s_bits[8];
  float acc[NC];
#pragma unroll
  for (int k = 0; k < NC; k++) acc[k] = 0.f;
  if (v == V) {                                          // the start token: every row of step 0
    for (int b = 0; b < B; b++)
#pragma unroll
      for (int k = 0; k < NC; k++)
        if (j0 + k * 256 < G) acc[k] += dz[(int64_t)b * G + j0 + k * 256];
  } else {
    const int total = B * (Tn - 1);                        // idx = (t - 1) B + b, t >= 1
    for (int base = 0; base < total; base += 256) {
      const int idx = base + threadIdx.x;
      bool hit = false;
      if (idx < total) {
        int64_t tk = formula[(int64_t)(idx % B) * f_stride + idx / B];
        if (tk < 0) tk = 0;
        if (tk >= V) tk = V - 1;
        hit = tk == (int64_t)v;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      if ((threadIdx.x & 31) == 0) s_bits[threadIdx.x >> 5] = bal;
      __syncthreads();
#pragma unroll
      for (int w = 0; w < 8; w++) {
        unsigned bits = s_bits[w];
        while (bits) {                                     // ascending index order -> deterministic sum
          const int k = __ffs(bits) - 1;
          bits &= bits - 1;
          const float* row = dz + ((int64_t)B + base + w * 32 + k) * G;      // row (t, b) of dz = B + idx
#pragma unroll
          for (int q = 0; q < NC; q++)
            if (j0 + q * 256 < G) acc[q] += row[j0 + q * 256];
        }
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int k = 0; k < NC; k++)
    if (j0 + k * 256 < G) dptab[(int64_t)v * G + j0 + k * 256] = acc[k];
}

// ------------------------------------------------------------------------------------------------ workspace
struct TfDims {
  int B, T, R, C, A, D, O, E, V, XH, G, LW, N2, DW, Vl, rpi, nimg;
};
static inline TfDims tf_dims(const lo_tfdec_args* a) {
  TfDims d;
  d.B = a->B; d.T = a->T; d.R = a->R; d.C = a->C; d.A = a->A; d.D = a->D; d.O = a->O; d.E = a->E; d.V = a->V;
  d.XH = a->O + a->D; d.G = 4 * a->D; d.LW = a->E + a->O + a->D; d.N2 = a->A + a->O; d.DW = a->A + a->O;
  d.Vl = a->ldl > 0 ? a->ldl : a->V;
  d.rpi = a->rows_per_img > 1 ? a->rows_per_img : 1;
  d.nimg = a->B / d.rpi;
  return d;
}

struct TfWs {
  void *att_img, *datt_img;                       // dt [nimg*R][A]
  float *dbeta_acc, *ptab, *dptab;
  float *xh, *call, *gates, *ztmp, *out2, *ctx, *oc, *dologit, *dout2, *dhc, *dz, *dxh, *dc, *de, *dctx, *mean, *initpre, *sinit,
      *dinit, *dmean, *dlogits, *row_loss, *gtmp, *hd, *sreg;
  bf16 *xh_bf, *ctx_bf, *dout2_bf, *dz_bf, *dlogits_bf, *hd_bf;
  void *wb4, *wb5, *wb6, *wbY, *wimgT;            // dt: transposed weights for the backward GEMMs
  void* attwork;
  void* ragmap;                                   // ragged decode (reg_off): CTA map and ticket counters of the attention launch
  int64_t* next_tok;
  int32_t *finished, *parent_rows;
  size_t bytes;
};

static TfWs tf_carve(const lo_tfdec_args* a) {
  const TfDims d = tf_dims(a);
  const size_t es = a->dt == LO_F32 ? 4 : 2;
  const bool bf = a->dt == LO_BF16;
  char* base = (char*)a->ws;
  size_t off = 0;
  auto take = [&](size_t bytes) -> void* {
    void* p = base ? base + off : nullptr;
    off += (bytes + 255) & ~(size_t)255;
    return p;
  };
  const size_t TB = (size_t)d.T * d.B, T1B = (size_t)(d.T + 1) * d.B;
  TfWs w{};
  w.att_img = take((size_t)d.nimg * d.R * d.A * es);
  w.datt_img = take((size_t)d.nimg * d.R * d.A * es);
  w.dbeta_acc = (float*)take((size_t)d.B * d.A * 4);
  w.ptab = (float*)take((size_t)(d.V + 1) * d.G * 4);
  w.dptab = (float*)take((size_t)(d.V + 1) * d.G * 4);
  w.xh = (float*)take(T1B * d.XH * 4);
  w.call = (float*)take(T1B * d.D * 4);
  w.gates = (float*)take(TB * d.G * 4);
  w.ztmp = (float*)take((size_t)d.B * d.G * 4);
  w.out2 = (float*)take(TB * d.N2 * 4);
  w.ctx = (float*)take(TB * d.C * 4);
  w.oc = (float*)take((size_t)d.B * d.O * 4);
  w.dologit = (float*)take(TB * d.O * 4);
  w.dout2 = (float*)take(TB * d.DW * 4);
  w.dhc = (float*)take((size_t)d.B * (d.D + d.C) * 4);
  w.dz = (float*)take(TB * d.G * 4);
  w.dxh = (float*)take((size_t)d.B * d.XH * 4);
  w.dc = (float*)take((size_t)d.B * d.D * 4);
  w.de = (float*)take((size_t)d.B * d.T * d.R * 4);
  w.dctx = (float*)take(TB * d.C * 4);
  w.mean = (float*)take((size_t)d.B * d.C * 4);
  w.initpre = (float*)take((size_t)d.B * (2 * d.D + d.O) * 4);
  w.sinit = (float*)take((size_t)d.B * (2 * d.D + d.O) * 4);
  w.dinit = (float*)take((size_t)d.B * (2 * d.D + d.O) * 4);
  w.dmean = (float*)take((size_t)d.B * d.C * 4);
  w.dlogits = (float*)take(TB * d.Vl * 4);
  w.row_loss = (float*)take(TB * 4);
  w.gtmp = (float*)take((size_t)d.B * (d.XH > d.D ? d.XH : d.D) * 4);
  w.xh_bf = bf ? (bf16*)take(T1B * d.XH * 2) : nullptr;
  w.ctx_bf = bf ? (bf16*)take(TB * d.C * 2) : nullptr;
  w.dout2_bf = bf ? (bf16*)take(TB * d.DW * 2) : nullptr;
  w.dz_bf = bf ? (bf16*)take(TB * d.G * 2) : nullptr;
  w.dlogits_bf = bf ? (bf16*)take(TB * d.Vl * 2) : nullptr;
  w.hd = (float*)take(TB * d.D * 4);                                  // dropped h_t (attention_cell.py:72), used when keep_h != NULL
  w.hd_bf = bf ? (bf16*)take(TB * d.D * 2) : nullptr;
  w.wb4 = take((size_t)(d.D + d.C) * d.O * es);
  w.wb5 = take((size_t)d.D * d.A * es);
  w.wb6 = take((size_t)d.XH * d.G * es);
  w.wbY = take((size_t)d.O * d.Vl * es);
  w.wimgT = take((size_t)d.C * d.A * es);
  w.attwork = take((size_t)lo_attention_workspace_bytes(d.B, d.C));
  w.next_tok = (int64_t*)take((size_t)d.B * 8);
  w.finished = (int32_t*)take((size_t)d.B * 4);
  w.parent_rows = (int32_t*)take((size_t)d.B * 4);
  w.sreg = (float*)take(TB * 4);                                      // generic backward: [B][T] sum_r alpha d alpha
  w.ragmap = take((size_t)attention_ragged_map_bytes(d.B));
  w.bytes = off;
  return w;
}

static int tf_check(const lo_tfdec_args* a, bool decode) {
  LO_CHECK_ARG(a != nullptr, "null args");
  LO_CHECK_ARG(a->B > 0 && a->B <= 512 && a->T > 0 && a->R > 0 && a->V > 1, "B in 1..512, T, R > 0, V > 1");
  LO_CHECK_ARG(a->C == 256 || a->C == 512 || a->C == 1024, "channels in {256,512,1024}");
  LO_CHECK_ARG(a->A == a->C || (a->A == 256 && a->C == 512), "(dim_e, channels): equal, or (256, 512) — the instantiated attention widths");
  LO_CHECK_ARG(a->D % 8 == 0 && a->O % 8 == 0 && a->E % 8 == 0, "num_units, dim_o, dim_embeddings multiples of 8");
  LO_CHECK_ARG(a->dt == LO_F32 || a->dt == LO_BF16, "dt");
  LO_CHECK_ARG(a->ldl == 0 || (a->ldl >= a->V && a->ldl % 8 == 0), "ldl >= V, multiple of 8");
  LO_CHECK_ARG(a->enc && a->ws && a->logits && a->alphas, "null buffer");
  LO_CHECK_ARG(a->w_img && a->w_cat2 && a->beta && a->w_lstm && a->b_lstm && a->w_oc && a->w_y && a->w_init && a->b_init && a->emb,
               "null parameter");
  const int rpi = a->rows_per_img > 1 ? a->rows_per_img : 1;
  LO_CHECK_ARG(a->B % rpi == 0, "B must be a multiple of rows_per_img");
  LO_TRY(check_reg_off(a, decode));
  if (decode) {
    LO_CHECK_ARG(!a->ss_prob && !a->fed && !a->ss_u && !a->ss_temp && !a->ss_gu && !a->ss_state,
                 "scheduled sampling (ss_prob, fed, ss_u, ss_temp, ss_gu, ss_state) is a training mode: greedy decode feeds its own "
                 "argmax already and beam search has no such mode");
  } else if (a->ss_prob) {
    LO_CHECK_ARG(a->fed, "scheduled sampling (ss_prob) needs fed");
    LO_CHECK_ARG(a->ss_u || a->ss_state, "scheduled sampling (ss_prob) needs ss_u or ss_state for its coin");
    LO_CHECK_ARG(rpi == 1, "scheduled sampling (ss_prob) needs rows_per_img <= 1");
    LO_CHECK_ARG(!a->ss_gu || a->ss_temp, "ss_gu (injected Gumbel uniforms) needs ss_temp");
  } else {
    LO_CHECK_ARG(!a->ss_temp && !a->ss_gu, "ss_temp / ss_gu (sampling with a temperature) need ss_prob");
  }
  LO_CHECK_ARG(g_opt_att_pipe, "the Genthial cell runs on the TMA-ring attention kernels only (option att_pipe=1)");
  return LO_OK;
}

// activations live in fp32 with a bf16 mirror (bf16 mode): C (+)= A W^T through the dispatcher (mma.sync kernel for M <= 64,
// wgmma otherwise, CUDA cores when the shape does not qualify)
static int tf_nt(const lo_tfdec_args* a, const float* A32, const bf16* Abf, int64_t lda, const void* W, int64_t ldw, float* C,
                 int64_t ldc, int M, int N, int K, const float* bias, int acc, cudaStream_t st) {
  if (a->dt == LO_BF16 && Abf && a->impl == LO_IMPL_TC)
    return gemm_nt(Abf, LO_BF16, lda, W, LO_BF16, ldw, C, LO_F32, ldc, M, N, K, bias, acc, 0, LO_IMPL_TC, st);
  return gemm_nt(A32, LO_F32, lda, W, a->dt, ldw, C, LO_F32, ldc, M, N, K, bias, acc, 0, LO_IMPL_SIMT, st);
}
// C[M][N] = A[K][M]^T B[K][N]   (hoisted weight gradients; wgmma when both operands have bf16 mirrors)
static int tf_tn(const lo_tfdec_args* a, const float* A32, const bf16* Abf, int64_t lda, const float* B32, const bf16* Bbf,
                 int64_t ldb, float* C, int64_t ldc, int M, int N, int K, cudaStream_t st) {
  if (a->dt == LO_BF16 && a->impl == LO_IMPL_TC && Abf && Bbf && tc_available() && lda % 8 == 0 && ldb % 8 == 0 &&
      ((uintptr_t)Abf & 15) == 0 && ((uintptr_t)Bbf & 15) == 0 && M >= 64 && N >= 64) {
    LO_CUDA(cudaMemset2DAsync(C, (size_t)ldc * 4, 0, (size_t)N * 4, (size_t)M, st));
    return tc_gemm_tn(Abf, lda, Bbf, ldb, C, ldc, M, N, K, st);
  }
  if (A32 && B32) return gemm_tn(A32, LO_F32, lda, B32, LO_F32, ldb, C, LO_F32, ldc, M, N, K, 0, LO_IMPL_SIMT, st);
  return gemm_tn(A32 ? (const void*)A32 : (const void*)Abf, A32 ? LO_F32 : LO_BF16, lda, B32 ? (const void*)B32 : (const void*)Bbf,
                 B32 ? LO_F32 : LO_BF16, ldb, C, LO_F32, ldc, M, N, K, 0, LO_IMPL_SIMT, st);
}

static int tf_prologue(const lo_tfdec_args* a, const TfDims& d, const TfWs& w, cudaStream_t st) {
  const int dt = a->dt;
  // att_img = img W_img, no bias, once (attention_mechanism.py:43); packed layout (reg_off): every region of every image once
  const int enc_rows = a->reg_off_host ? a->reg_off_host[d.nimg] : d.nimg * d.R;
  LO_TRY(gemm_nt(a->enc, dt, d.C, a->w_img, dt, d.C, w.att_img, dt, d.A, enc_rows, d.A, d.C, nullptr, 0, 0, a->impl, st));
  // token -> gate pre-activation table: [embedding_table ; start_token] K[:E] + b   (replaces the lookup + x[:, :E] K[:E])
  LO_TRY(gemm_nt(a->emb, dt, d.E, a->w_lstm, dt, d.LW, w.ptab, LO_F32, d.G, d.V + 1, d.G, d.E, a->b_lstm, 0, 0, LO_IMPL_SIMT, st));
  {
    dim3 grid(cdiv(d.C, 256), d.B);
    if (a->reg_off)
      LO_DISPATCH_DT(dt, T, (mean_segments_kernel<T><<<grid, 256, 0, st>>>((const T*)a->enc, w.mean, a->reg_off, d.C, d.rpi)));
    else
      LO_DISPATCH_DT(dt, T, (mean_rows_kernel<T><<<grid, 256, 0, st>>>((const T*)a->enc, w.mean, d.R, d.C, d.rpi)));
    LO_LAUNCH_OK();
  }
  const int IW = 2 * d.D + d.O;
  LO_TRY(gemm_nt(w.mean, LO_F32, d.C, a->w_init, dt, d.C, w.initpre, LO_F32, IW, d.B, IW, d.C, a->b_init, 0, 0, LO_IMPL_SIMT, st));
  tf_init_state_kernel<<<cdiv((long)d.B * IW, 256), 256, 0, st>>>(w.initpre, w.sinit, w.call, w.xh, w.xh_bf, d.XH, d.B, d.D, d.O);
  LO_LAUNCH_OK();
  return LO_OK;
}

// one cell step: consumes xh[t] = [o_{t-1} | h_{t-1}], call[t]; produces xh[t+1], call[t+1], alphas[:, t], ctx[t].  rg: decode with
// per-image region counts (the ragged attention launch), NULL otherwise
// the sampling operands of the pointwise kernel that chooses fed[:, ti] from the logits of step ti (lo_tfdec_args.ss_prob)
static SsStep tf_ss_step(const lo_tfdec_args* a, const TfDims& d, int ti) {
  SsStep ss{};
  ss.prev_logits = a->logits + (int64_t)ti * d.B * d.Vl;      // time-major: row b of step ti
  ss.lstride = d.Vl;
  ss.prob = a->ss_prob;
  ss.u = a->ss_u ? a->ss_u + ti : nullptr;
  ss.coin_state = (const unsigned long long*)a->ss_state;
  ss.ustride = d.T;
  ss.fed = a->fed + ti;
  return ss;
}
static GumbelStep tf_gumbel_step(const lo_tfdec_args* a, const TfDims& d, int ti) {
  return GumbelStep{a->ss_temp, a->ss_gu ? a->ss_gu + (int64_t)ti * d.V : nullptr, (int64_t)d.T * d.V};
}

static int tf_step(const lo_tfdec_args* a, const TfDims& d, const TfWs& w, int t, const int64_t* tok, int64_t tok_stride,
                   cudaStream_t st, const AttRagged* rg = nullptr) {
  const size_t es = a->dt == LO_F32 ? 4 : 2;
  const int64_t rowt = (int64_t)t * d.B, rown = (int64_t)(t + 1) * d.B;
  const float* xh_t = w.xh + rowt * d.XH;
  float* xh_n = w.xh + rown * d.XH;
  const bf16* xhb_t = w.xh_bf ? w.xh_bf + rowt * d.XH : nullptr;
  bf16* xhb_n = w.xh_bf ? w.xh_bf + rown * d.XH : nullptr;
  float* out2 = w.out2 + rowt * d.N2;
  // z = [o_{t-1} ; h_{t-1}] K[E:]   (attention_cell.py:70-71; the embedding rows of K come from the table)
  LO_TRY(tf_nt(a, xh_t, xhb_t, d.XH, (const char*)a->w_lstm + (size_t)d.E * es, d.LW, w.ztmp, d.G, d.B, d.G, d.XH, nullptr, 0, st));
  // the pointwise launch; `extra`: the step index and sampling operands of tf_lstm_pw_fwd_ss_kernel
  auto launch_pw = [&](auto kernel, auto... extra) {
    return launch_pdl(kernel, dim3(cdiv((long)d.B * d.D, 256)), dim3(256), (size_t)0, st, (const float*)w.ztmp, (const float*)w.ptab, tok,
                      tok_stride, d.V, (const float*)(w.call + rowt * d.D), w.gates + rowt * d.G, w.call + rown * d.D, xh_n + d.O,
                      xhb_n ? xhb_n + d.O : (bf16*)nullptr, (int64_t)d.XH, a->keep_h ? a->keep_h + rowt * d.D : (const float*)nullptr,
                      w.hd + rowt * d.D, w.hd_bf ? w.hd_bf + rowt * d.D : (bf16*)nullptr, d.B, d.D, extra...);
  };
  if (a->ss_prob && t > 0)          // sampling: the token consumed now is chosen from the logits of step t-1
    LO_CUDA(launch_pw(a->ss_temp ? tf_lstm_pw_fwd_ss_kernel<2> : tf_lstm_pw_fwd_ss_kernel<1>, t - 1, tf_ss_step(a, d, t - 1),
                      tf_gumbel_step(a, d, t - 1)));
  else
    LO_CUDA(launch_pw(tf_lstm_pw_fwd_kernel));
  LO_LAUNCH_OK();
  // [hd_t W_h | hd_t o_W_h] with hd_t = dropout(h_t)   (attention_cell.py:72, attention_mechanism.py:79, attention_cell.py:82)
  if (a->keep_h)
    LO_TRY(tf_nt(a, w.hd + rowt * d.D, w.hd_bf ? w.hd_bf + rowt * d.D : nullptr, d.D, a->w_cat2, d.D, out2, d.N2, d.B, d.N2, d.D, nullptr, 0, st));
  else
    LO_TRY(tf_nt(a, xh_n + d.O, xhb_n ? xhb_n + d.O : nullptr, d.XH, a->w_cat2, d.D, out2, d.N2, d.B, d.N2, d.D, nullptr, 0, st));
  {
    AttFwdArgs x{w.att_img, a->enc, out2, d.N2, a->beta, a->alphas + (int64_t)t * d.R, (int64_t)d.T * d.R, w.ctx + rowt * d.C, nullptr,
                 0, nullptr, w.ctx_bf ? w.ctx_bf + rowt * d.C : nullptr, d.B, d.R, w.attwork, d.rpi, 1, d.A};
    if (rg)
      LO_TRY(attention_fwd_ragged(x, *rg, a->dt, d.C, st));
    else
      LO_TRY(attention_fwd_pipe(x, a->dt, d.C, st));
  }
  // o_t = tanh(h_t o_W_h + ctx o_W_c)
  LO_TRY(tf_nt(a, w.ctx + rowt * d.C, w.ctx_bf ? w.ctx_bf + rowt * d.C : nullptr, d.C, a->w_oc, d.C, w.oc, d.O, d.B, d.O, d.C, nullptr, 0,
               st));
  LO_CUDA(launch_pdl(tf_o_pw_fwd_kernel, dim3(cdiv((long)d.B * d.O, 256)), dim3(256), (size_t)0, st, (const float*)w.oc,
                     (const float*)(out2 + d.A), (int64_t)d.N2, a->keep_o ? a->keep_o + rowt * d.O : (const float*)nullptr, xh_n, xhb_n,
                     (int64_t)d.XH, d.B, d.O));
  LO_LAUNCH_OK();
  return LO_OK;
}

// logits of `rows` consecutive state rows starting at xh row `row0` (o part) -> out [rows][ldo]
static int tf_logits(const lo_tfdec_args* a, const TfDims& d, const TfWs& w, int64_t row0, int rows, float* out, int64_t ldo,
                     cudaStream_t st) {
  return tf_nt(a, w.xh + row0 * d.XH, w.xh_bf ? w.xh_bf + row0 * d.XH : nullptr, d.XH, a->w_y, d.O, out, ldo, rows, d.V, d.O, nullptr, 0,
               st);
}

// the TF flavour in the decode loops of lo_decoder.cu: its scratch, the ragged CTA map included, is carved from ws
struct TfDecode {
  const lo_tfdec_args* a;
  TfDims d;
  TfWs w;
  DecodeCtx c;
  explicit TfDecode(const lo_tfdec_args* a_)
      : a(a_), d(tf_dims(a_)), w(tf_carve(a_)),
        c{d.B, d.T, d.V, d.rpi, a_->logits, w.next_tok, w.finished, w.parent_rows,
          AttRagged{a_->reg_off, a_->reg_off_host, w.ragmap, 0}} {}
  int prologue(cudaStream_t st) { return tf_prologue(a, d, w, st); }
  // step 0 is fed tok = NULL: the start-token row V of the token table
  int step(int t, cudaStream_t st) {
    LO_TRY(tf_step(a, d, w, t, t == 0 ? nullptr : w.next_tok, 1, st, c.ragged()));
    return tf_logits(a, d, w, (int64_t)(t + 1) * d.B, d.B, a->logits, d.V, st);
  }
  // the cell state (c, h, o) of step t by parents (gather_helper, beam_search_decoder_cell.py:370-391): xh and its mirror, then c
  int reorder(int t, cudaStream_t st) {
    const int64_t rown = (int64_t)(t + 1) * d.B;
    gather_rows_kernel<<<cdiv((long)d.B * d.XH, 256), 256, 0, st>>>(w.xh + rown * d.XH, c.parent_rows, w.gtmp,
                                                                    w.xh_bf ? w.xh_bf + rown * d.XH : nullptr, d.B, d.XH);
    LO_LAUNCH_OK();
    LO_CUDA(cudaMemcpyAsync(w.xh + rown * d.XH, w.gtmp, (size_t)d.B * d.XH * 4, cudaMemcpyDeviceToDevice, st));
    gather_rows_kernel<<<cdiv((long)d.B * d.D, 256), 256, 0, st>>>(w.call + rown * d.D, c.parent_rows, w.gtmp, nullptr, d.B, d.D);
    LO_LAUNCH_OK();
    LO_CUDA(cudaMemcpyAsync(w.call + rown * d.D, w.gtmp, (size_t)d.B * d.D * 4, cudaMemcpyDeviceToDevice, st));
    return LO_OK;
  }
};

}  // namespace lo

using namespace lo;

extern "C" {

int64_t lo_sizeof_tfdec_args(void) { return (int64_t)sizeof(lo_tfdec_args); }

int64_t lo_tfdec_workspace_bytes(const lo_tfdec_args* a) {
  if (!a) return 0;
  lo_tfdec_args tmp = *a;
  tmp.ws = nullptr;
  return (int64_t)tf_carve(&tmp).bytes;
}

int lo_tfdec_forward(const lo_tfdec_args* a, int with_loss, void* stream) {
  LO_TRY(tf_check(a, false));
  LO_CHECK_ARG(a->formula && a->formula_stride >= a->T, "formula [B][>= T]");
  LO_CHECK_ARG(!with_loss || (a->lengths && a->loss && a->inv_n_words > 0.f), "lengths / loss / inv_n_words");
  cudaStream_t st = (cudaStream_t)stream;
  const TfDims d = tf_dims(a);
  LO_CHECK_ARG(d.rpi == 1, "training runs with rows_per_img = 1");
  const TfWs w = tf_carve(a);
  LO_TRY(tf_prologue(a, d, w, st));
  const bool sampling = a->ss_prob != nullptr;
  for (int t = 0; t < d.T; t++) {
    LO_TRY(tf_step(a, d, w, t, t == 0 ? nullptr : a->formula + (t - 1), a->formula_stride, st));
    // sampling: the head of step t inside the loop (the next step's cell chooses its token from these logits)
    if (sampling) LO_TRY(tf_logits(a, d, w, (int64_t)(t + 1) * d.B, d.B, a->logits + (int64_t)t * d.B * d.Vl, d.Vl, st));
  }
  if (sampling) {
    // fed[:, T-1]: chosen like the others, consumed by no step.  One warp per row (the block geometry of a row width of 32)
    const SsStep ss = tf_ss_step(a, d, d.T - 1);
    const GumbelStep gs = tf_gumbel_step(a, d, d.T - 1);
    const int64_t* tok = a->formula + (d.T - 1);
    const dim3 grid(cdiv((long)d.B * 32, 256));
    if (a->ss_temp)
      tf_ss_last_token_kernel<2><<<grid, 256, 0, st>>>(tok, a->formula_stride, d.V, d.B, 32, d.T - 1, ss, gs);
    else
      tf_ss_last_token_kernel<1><<<grid, 256, 0, st>>>(tok, a->formula_stride, d.V, d.B, 32, d.T - 1, ss, gs);
    LO_LAUNCH_OK();
  } else {
    // logits for all (t, b) in one GEMM: rows 1..T of xh hold o_t   (attention_cell.py:84)
    LO_TRY(tf_logits(a, d, w, d.B, d.T * d.B, a->logits, d.Vl, st));
  }
  if (!with_loss) return LO_OK;
  const int rows = d.T * d.B;
  tf_ce_kernel<<<cdiv(rows, 8), 256, 0, st>>>(a->logits, a->formula, a->formula_stride, a->lengths, w.row_loss, w.dlogits, w.dlogits_bf,
                                              d.B, d.T, d.V, d.Vl, a->inv_n_words);
  LO_LAUNCH_OK();
  loss_finalize_kernel<<<1, 1024, 0, st>>>(w.row_loss, rows, nullptr, 0, a->inv_n_words, 0.f, a->loss);
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_tfdec_backward(const lo_tfdec_args* a, void* stream) {
  LO_TRY(tf_check(a, false));
  LO_CHECK_ARG(a->dlogits_ext || !a->dalpha_ext, "dalpha_ext needs dlogits_ext (generic mode)");
  LO_CHECK_ARG(!a->dlogits_ext || a->dlogits_stride >= a->V, "dlogits_stride >= V");
  LO_CHECK_ARG(a->formula && a->denc, "formula / denc");
  LO_CHECK_ARG(a->g_w_img && a->g_w_cat2 && a->g_beta && a->g_w_lstm && a->g_b_lstm && a->g_w_oc && a->g_w_y && a->g_w_init &&
                   a->g_b_init && a->g_emb, "null gradient buffer");
  cudaStream_t st = (cudaStream_t)stream;
  const TfDims d = tf_dims(a);
  const TfWs w = tf_carve(a);
  const int dt = a->dt;
  const int TB = d.T * d.B;
  const dim3 tb(32, 8);
  // generic mode: d logits from the caller (batch-major -> the time-major workspace rows; every position carries gradient), and
  // sreg[b,t] = sum_r alpha d alpha for the attention backward.  Plain launches: everything after them waits for them.
  if (a->dlogits_ext) {
    const bool bf_mirror = dt == LO_BF16 && a->impl == LO_IMPL_TC;            // the wgmma GEMMs read d logits in bf16 (tf_nt / tf_tn)
    dpred_kernel<<<dim3(cdiv(d.Vl, 128), (unsigned)(TB < 65535 ? TB : 65535)), 128, 0, st>>>(
        a->dlogits_ext, a->dlogits_stride, nullptr, w.dlogits, bf_mirror ? w.dlogits_bf : nullptr, d.T, d.V, d.Vl, (int64_t)TB, d.B);
    LO_LAUNCH_OK();
    if (a->dalpha_ext) {
      sreg_kernel<<<cdiv(TB, 8), 256, 0, st>>>(a->alphas, a->dalpha_ext, (int64_t)d.T * d.R, d.R, w.sreg, d.B, d.T, d.R);
      LO_LAUNCH_OK();
    }
  }
  const float* dal = a->dalpha_ext;          // d alpha rows [B][T][R] (generic mode only, checked above) or none
  // transposed shadows for the backward GEMMs (dX = dY W needs W as [in][out] = the TF layout); out[n][k] = in[k][n]
  auto transpose = [&](const void* in, int64_t off_in, int64_t ld_in, void* out, int64_t off_out, int64_t ld_out, int K, int N) -> int {
    LO_DISPATCH_DT(dt, T, (transpose_kernel<T><<<dim3(cdiv(N, 32), cdiv(K, 32)), tb, 0, st>>>((const T*)in + off_in, ld_in, (T*)out + off_out,
                                                                                                ld_out, K, N)));
    LO_LAUNCH_OK();
    return LO_OK;
  };
  LO_TRY(transpose(a->w_cat2, (int64_t)d.A * d.D, d.D, w.wb4, 0, d.O, d.O, d.D));             // o_W_h^T [O][D] -> [D][O]
  LO_TRY(transpose(a->w_oc, 0, d.C, w.wb4, (int64_t)d.D * d.O, d.O, d.O, d.C));               // o_W_c^T [O][C] -> [C][O]
  LO_TRY(transpose(a->w_cat2, 0, d.D, w.wb5, 0, d.A, d.A, d.D));                              // att_h^T [A][D] -> [D][A]
  LO_TRY(transpose(a->w_lstm, d.E, d.LW, w.wb6, 0, d.G, d.G, d.XH));                          // K[E:]^T [4D][O+D] -> [O+D][4D]
  LO_TRY(transpose(a->w_y, 0, d.O, w.wbY, 0, d.Vl, d.V, d.O));                                // y_W_o^T [V][O] -> [O][Vl]
  LO_TRY(transpose(a->w_img, 0, d.C, w.wimgT, 0, d.A, d.A, d.C));                             // W_img^T [A][C] -> [C][A]
  // d o (logit path) for every step at once: dlogits @ y_W_o^T
  LO_TRY(tf_nt(a, w.dlogits, w.dlogits_bf, d.Vl, w.wbY, d.Vl, w.dologit, d.O, TB, d.O, d.Vl, nullptr, 0, st));
  LO_CUDA(cudaMemsetAsync(w.dxh, 0, (size_t)d.B * d.XH * 4, st));
  LO_CUDA(cudaMemsetAsync(w.dc, 0, (size_t)d.B * d.D * 4, st));
  LO_CUDA(cudaMemsetAsync(w.dbeta_acc, 0, (size_t)d.B * d.A * 4, st));
  for (int t = d.T - 1; t >= 0; t--) {
    const int64_t rowt = (int64_t)t * d.B, rown = (int64_t)(t + 1) * d.B;
    float* dout2 = w.dout2 + rowt * d.DW;
    bf16* dout2b = w.dout2_bf ? w.dout2_bf + rowt * d.DW : nullptr;
    LO_CUDA(launch_pdl(tf_o_pw_bwd_kernel, dim3(cdiv((long)d.B * d.O, 256)), dim3(256), (size_t)0, st, w.dxh, (int64_t)d.XH,
                       (const float*)(w.dologit + rowt * d.O), a->keep_o ? a->keep_o + rowt * d.O : (const float*)nullptr,
                       (const float*)(w.xh + rown * d.XH), dout2 + d.A, dout2b ? dout2b + d.A : (bf16*)nullptr, (int64_t)d.DW, d.B, d.O));
    LO_LAUNCH_OK();
    // [d h_t (o path) | d ctx] = d pre_o [o_W_h^T | o_W_c^T]
    LO_TRY(tf_nt(a, dout2 + d.A, dout2b ? dout2b + d.A : nullptr, d.DW, w.wb4, d.O, w.dhc, d.D + d.C, d.B, d.D + d.C, d.O, nullptr, 0, st));
    {
      AttBwdArgs x{w.att_img, a->enc, w.out2 + rowt * d.N2, nullptr, d.N2, a->beta, a->alphas + (int64_t)t * d.R, (int64_t)d.T * d.R,
                   w.ctx + rowt * d.C, w.dhc + d.D, d.D + d.C, dal ? dal + (int64_t)t * d.R : nullptr, dal ? (int64_t)d.T * d.R : 0,
                   dal ? w.sreg + t : nullptr, dal ? d.T : 0, w.de + (int64_t)t * d.R, dout2, nullptr, d.DW,
                   dout2b, nullptr, w.dctx + rowt * d.C, d.B, d.R, w.attwork, w.dbeta_acc, 1, d.A};
      x.ordered_dwf = g_opt_det;
      LO_TRY(attention_bwd_pipe(x, dt, d.C, st));
    }
    // d h_t += d att_h W_h^T
    LO_TRY(tf_nt(a, dout2, dout2b, d.DW, w.wb5, d.A, w.dhc, d.D + d.C, d.B, d.D, d.A, nullptr, 1, st));
    LO_CUDA(launch_pdl(tf_lstm_pw_bwd_kernel, dim3(cdiv((long)d.B * d.D, 256)), dim3(256), (size_t)0, st, w.dxh, (int64_t)d.XH, d.O,
                       (const float*)w.dhc, (int64_t)(d.D + d.C), a->keep_h ? a->keep_h + rowt * d.D : (const float*)nullptr, w.dc,
                       (const float*)(w.gates + rowt * d.G), (const float*)(w.call + rowt * d.D), (const float*)(w.call + rown * d.D),
                       w.dz + rowt * d.G, w.dz_bf ? w.dz_bf + rowt * d.G : (bf16*)nullptr, d.B, d.D));
    LO_LAUNCH_OK();
    // [d o_{t-1} | d h_{t-1}] += d z K[E:]^T
    LO_TRY(tf_nt(a, w.dz + rowt * d.G, w.dz_bf ? w.dz_bf + rowt * d.G : nullptr, d.G, w.wb6, d.G, w.dxh, d.XH, d.B, d.XH, d.G, nullptr, 1, st));
  }
  // ---- hoisted parameter gradients (stacked over all T*B rows) ----
  // h_t as the attention / o projections saw it: rows 1..T of xh, or the dropped copies when dropout is on
  const float* H32 = a->keep_h ? w.hd : w.xh + (int64_t)d.B * d.XH + d.O;
  const bf16* Hbf = a->keep_h ? w.hd_bf : (w.xh_bf ? w.xh_bf + (int64_t)d.B * d.XH + d.O : nullptr);
  const int64_t ldH = a->keep_h ? d.D : d.XH;
  const float* O32 = w.xh + (int64_t)d.B * d.XH;                             // o_t
  const bf16* Obf = w.xh_bf ? w.xh_bf + (int64_t)d.B * d.XH : nullptr;
  // LSTM kernel, [o ; h] rows: dz^T xh[0..T-1]
  LO_TRY(tf_tn(a, w.dz, w.dz_bf, d.G, w.xh, w.xh_bf, d.XH, a->g_w_lstm + d.E, d.LW, d.G, d.XH, TB, st));
  // embedding rows through the table: d ptab (scatter, or the fixed-order gather under option deterministic), then d emb =
  // d ptab K[:E]^T..., d K[:E] = d ptab^T emb, d b = colsum (sampling: the tokens the forward fed, not the targets)
  {
    const int64_t* tok = a->ss_prob ? a->fed : a->formula;
    const int64_t tok_stride = a->ss_prob ? (int64_t)d.T : a->formula_stride;
    if (g_opt_det) {
      tf_dptab_kernel<<<dim3(cdiv(d.G, TF_DPT_COLS), d.V + 1), 256, 0, st>>>(w.dz, tok, tok_stride, w.dptab, d.B, d.T, d.G, d.V);
    } else {
      LO_CUDA(cudaMemsetAsync(w.dptab, 0, (size_t)(d.V + 1) * d.G * 4, st));
      tf_dptab_scatter_kernel<<<LO_NUM_SMS * 8, 256, 0, st>>>(w.dz, tok, tok_stride, w.dptab, d.B, d.T, d.G, d.V);
    }
  }
  LO_LAUNCH_OK();
  LO_TRY(gemm_nn(w.dptab, LO_F32, d.G, a->w_lstm, dt, d.LW, a->g_emb, LO_F32, d.E, d.V + 1, d.E, d.G, 0, LO_IMPL_SIMT, st));
  LO_TRY(gemm_tn(w.dptab, LO_F32, d.G, a->emb, dt, d.E, a->g_w_lstm, LO_F32, d.LW, d.G, d.E, d.V + 1, 0, LO_IMPL_SIMT, st));
  LO_TRY(colsum(w.dptab, LO_F32, a->g_b_lstm, d.V + 1, d.G, d.G, 0, st));
  // att_h.kernel and o_W_h (adjacent rows of w_cat2), o_W_c, y_W_o
  LO_TRY(tf_tn(a, w.dout2, w.dout2_bf, d.DW, H32, Hbf, ldH, a->g_w_cat2, d.D, d.A, d.D, TB, st));
  LO_TRY(tf_tn(a, w.dout2 + d.A, w.dout2_bf ? w.dout2_bf + d.A : nullptr, d.DW, H32, Hbf, ldH, a->g_w_cat2 + (int64_t)d.A * d.D, d.D, d.O,
               d.D, TB, st));
  LO_TRY(tf_tn(a, w.dout2 + d.A, w.dout2_bf ? w.dout2_bf + d.A : nullptr, d.DW, w.ctx, w.ctx_bf, d.C, a->g_w_oc, d.C, d.O, d.C, TB, st));
  LO_TRY(tf_tn(a, w.dlogits, w.dlogits_bf, d.Vl, O32, Obf, d.XH, a->g_w_y, d.O, d.V, d.O, TB, st));
  // att_beta: per-row partial sums were accumulated by the attention backward kernels
  LO_TRY(colsum(w.dbeta_acc, LO_F32, a->g_beta, d.B, d.A, d.A, 0, st));
  // d att_img[b,r,a] = beta[a] sum_t de[b,t,r] (1 - tanh^2(att_img + att_h_t))   (one sweep over t)
  {
    dim3 grid(d.A / 64, cdiv(d.R, 32), d.B);
    LO_DISPATCH_DT(dt, T, (datt1_kernel<T, 0, 1><<<grid, 128, 0, st>>>((const T*)w.att_img, w.out2, d.N2, (int64_t)d.B * d.N2, w.de, a->beta,
                                                                            (T*)w.datt_img, nullptr, d.T, d.R, d.A, 1, 0)));
    LO_LAUNCH_OK();
  }
  const int BR = d.B * d.R;
  // att_img.kernel: d W_img^T [A][C] = d att_img^T enc ; d enc = d att_img W_img^T
  if (dt == LO_BF16) {
    LO_TRY(tf_tn(a, nullptr, (const bf16*)w.datt_img, d.A, nullptr, (const bf16*)a->enc, d.C, a->g_w_img, d.C, d.A, d.C, BR, st));
    LO_TRY(gemm_nt(w.datt_img, LO_BF16, d.A, w.wimgT, LO_BF16, d.A, a->denc, LO_F32, d.C, BR, d.C, d.A, nullptr, 0, 0, a->impl, st));
  } else {
    LO_TRY(gemm_tn(w.datt_img, LO_F32, d.A, a->enc, LO_F32, d.C, a->g_w_img, LO_F32, d.C, d.A, d.C, BR, 0, LO_IMPL_SIMT, st));
    LO_TRY(gemm_nn(w.datt_img, LO_F32, d.A, a->w_img, LO_F32, d.C, a->denc, LO_F32, d.C, BR, d.C, d.A, 0, LO_IMPL_SIMT, st));
  }
  // d enc[b] += alphas[b]^T dctx[:, b, :]   (the context read, summed over time)
  {
    GemmDesc g{d.R, d.C, d.T, 1, d.R, (int64_t)d.B * d.C, 1, d.C, d.B, (int64_t)d.T * d.R, d.C, (int64_t)d.R * d.C, nullptr, 1, 0};
    LO_TRY(gemm(a->alphas, LO_F32, w.dctx, LO_F32, a->denc, LO_F32, g, LO_IMPL_SIMT, st));
  }
  // initial states: d(c0,h0,o0) -> tanh -> W_*_0, b_*_0, mean -> d enc
  const int IW = 2 * d.D + d.O;
  tf_init_bwd_kernel<<<cdiv((long)d.B * IW, 256), 256, 0, st>>>(w.dc, w.dxh, d.XH, w.sinit, w.dinit, d.B, d.D, d.O);
  LO_LAUNCH_OK();
  LO_TRY(gemm_tn(w.dinit, LO_F32, IW, w.mean, LO_F32, d.C, a->g_w_init, LO_F32, d.C, IW, d.C, d.B, 0, LO_IMPL_SIMT, st));
  LO_TRY(colsum(w.dinit, LO_F32, a->g_b_init, d.B, IW, IW, 0, st));
  LO_TRY(gemm_nn(w.dinit, LO_F32, IW, a->w_init, dt, d.C, w.dmean, LO_F32, d.C, d.B, d.C, IW, 0, LO_IMPL_SIMT, st));
  {
    const int64_t total = (int64_t)d.B * d.R * d.C;
    add_rowbcast_kernel<<<LO_NUM_SMS * 8, 256, 0, st>>>(a->denc, w.dmean, d.R, d.C, 1.0f / (float)d.R, total);
    LO_LAUNCH_OK();
  }
  return LO_OK;
}

int lo_tfdec_greedy(const lo_tfdec_args* a, int64_t end_id, int max_steps, int64_t* tokens, int32_t* fin_hist, void* stream) {
  LO_TRY(tf_check(a, true));
  TfDecode f(a);
  return greedy_loop(f, end_id, max_steps, tokens, fin_hist, (cudaStream_t)stream);
}

int lo_tfdec_beam(const lo_tfdec_args* a, int64_t end_id, int max_steps, int64_t* ids, int64_t* parents, int32_t* fin_hist, float* logp,
                  void* stream) {
  return lo_tfdec_beam_div(a, end_id, max_steps, ids, parents, fin_hist, logp, 1.f, 0.f, nullptr, nullptr, stream);
}

int lo_tfdec_beam_div(const lo_tfdec_args* a, int64_t end_id, int max_steps, int64_t* ids, int64_t* parents, int32_t* fin_hist,
                      float* logp, float div_gamma, float div_prob, const float* div_u, const uint64_t* div_state, void* stream) {
  LO_TRY(tf_check(a, true));
  TfDecode f(a);
  return beam_loop(f, BeamArgs{f.d.rpi, div_gamma, div_prob, div_u, div_state}, end_id, max_steps, ids, parents, fin_hist, logp,
                   (cudaStream_t)stream);
}

}  // extern "C"
