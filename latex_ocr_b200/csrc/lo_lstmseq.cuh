// Generic sequence LSTM (nn.LSTM / nn.LSTMCell semantics, gate order i,f,g,o, two bias vectors): forward over S steps for M
// independent sequences and the hand-derived backward.  EXTENSION beyond the reference (BASELINE.json configs[3]: row-encoder
// biLSTM over the CNN feature rows + a second decoder layer; the reference only links the paper, model/decoder.py:16): there is no
// reference code to restate — the oracle is torch.nn.LSTM itself (oracle/ref_ext.py).  Part of the lo_decoder.cu translation unit
// (reuses its transpose / cast kernels and the GEMM dispatcher: wgmma for the hoisted products and the M > 64 per-step
// projections, the mma.sync kernel for M <= 64, CUDA cores in fp32 mode).
//
// Schedule (same ideas as the decoder, DESIGN.md §4): the input projection x W_ih^T + b of ALL steps is one hoisted GEMM; the time
// loop is h_{p-1} W_hh^T (accumulated onto the hoisted pre-activations) + one pointwise cell kernel per step; every weight
// gradient and d x are GEMMs over the stacked per-step quantities after the loop.  Internally everything is dense and ordered
// by PROCESSING step p (p = t, or S-1-t for the reverse direction of a bidirectional layer); the caller's layouts (any row /
// step strides, e.g. the [N][H'][W'][C] feature map read row by row) are converted by a gather before and a scatter after.

namespace lo {

struct SeqDims { int S, M, I, H, G; };

struct SeqWs {
  void* xt;                 // dt  [S][M][I]   inputs in processing order
  float* gates;             // f32 [S][M][4H]  hoisted pre-activations, then post-activation gates
  float* h; float* c;       // f32 [S+1][M][H]
  bf16* h_bf;               // bf16 mirror of h (bf16 mode)
  float* dG; bf16* dG_bf;   // f32 [S][M][4H] (+ bf16 mirror)
  float* dh; float* dc;     // f32 [M][H] carried gradients
  float* dxt;               // f32 [S][M][I]
  void* whhT; void* wihT;   // dt [H][4H], [I][4H]
  float* bsum;              // f32 [4H] = b_ih + b_hh
  size_t bytes;
};

static SeqWs seq_carve(const lo_lstm_seq_args* a) {
  const size_t es = a->dt == LO_F32 ? 4 : 2;
  const bool bf = a->dt == LO_BF16;
  const size_t S = a->S, M = a->M, I = a->I, H = a->H, G = 4 * (size_t)a->H;
  char* base = (char*)a->ws;
  size_t off = 0;
  auto take = [&](size_t bytes) -> void* {
    void* p = base ? base + off : nullptr;
    off += (bytes + 255) & ~(size_t)255;
    return p;
  };
  SeqWs w{};
  w.xt = take(S * M * I * es);
  w.gates = (float*)take(S * M * G * 4);
  w.h = (float*)take((S + 1) * M * H * 4);
  w.c = (float*)take((S + 1) * M * H * 4);
  w.h_bf = bf ? (bf16*)take((S + 1) * M * H * 2) : nullptr;
  w.dG = (float*)take(S * M * G * 4);
  w.dG_bf = bf ? (bf16*)take(S * M * G * 2) : nullptr;
  w.dh = (float*)take(M * H * 4);
  w.dc = (float*)take(M * H * 4);
  w.dxt = (float*)take(S * M * I * 4);
  w.whhT = take(H * G * es);
  w.wihT = take(I * G * es);
  w.bsum = (float*)take(G * 4);
  w.bytes = off;
  return w;
}

// xt[p][m][:] = x[m * x_row + t(p) * x_step + :]  (storage dtype in, storage dtype out), 8 elements per thread
template <typename T>
__global__ void seq_gather_kernel(const T* __restrict__ x, int64_t x_row, int64_t x_step, T* __restrict__ xt, int S, int M, int I,
                                  int reverse) {
  const int64_t total = (int64_t)S * M * (I / 8);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % (I / 8));
    const int64_t pm = i / (I / 8);
    const int m = (int)(pm % M), p = (int)(pm / M);
    const int t = reverse ? S - 1 - p : p;
    float v[8];
    ld8(x + (int64_t)m * x_row + (int64_t)t * x_step + c8 * 8, v);
    st8(xt + pm * I + c8 * 8, v);
  }
}
// dx[m * x_row + t(p) * x_step + :] (+)= dxt[p][m][:]
__global__ void seq_scatter_kernel(const float* __restrict__ dxt, float* __restrict__ dx, int64_t x_row, int64_t x_step, int S, int M,
                                   int I, int reverse, int accumulate) {
  const int64_t total = (int64_t)S * M * (I / 4);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % (I / 4));
    const int64_t pm = i / (I / 4);
    const int m = (int)(pm % M), p = (int)(pm / M);
    const int t = reverse ? S - 1 - p : p;
    float4 v = *reinterpret_cast<const float4*>(dxt + pm * I + c4 * 4);
    float4* o = reinterpret_cast<float4*>(dx + (int64_t)m * x_row + (int64_t)t * x_step + c4 * 4);
    if (accumulate) { const float4 u = *o; v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w; }
    *o = v;
  }
}
__global__ void seq_bias_sum_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ o, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = a[i] + b[i];
}
// h0 / c0 (or zeros) into slot 0 (+ bf16 mirror of h)
__global__ void seq_init_kernel(const float* __restrict__ h0, const float* __restrict__ c0, float* __restrict__ h, float* __restrict__ c,
                                bf16* __restrict__ h_bf, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float hv = h0 ? h0[i] : 0.f;
  h[i] = hv;
  c[i] = c0 ? c0[i] : 0.f;
  if (h_bf) h_bf[i] = __float2bfloat16_rn(hv);
}

// the cell: gates (pre-activations, overwritten by the activations), c_prev -> c, h (+ bf16), and the caller's output tensors
__global__ void seq_lstm_pw_fwd_kernel(float* __restrict__ gates, const float* __restrict__ c_prev, float* __restrict__ c_out,
                                       float* __restrict__ h_out, bf16* __restrict__ h_bf, float* __restrict__ hs, void* __restrict__ hs_st,
                                       int st_is_bf16, int64_t hs_row, int M, int H) {
  pdl_wait();
  pdl_trigger();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * H) return;
  const int m = idx / H, j = idx % H;
  float* g = gates + (int64_t)m * 4 * H;
  const float i = sigmoidf_(g[j]), f = sigmoidf_(g[H + j]), gg = tanhf(g[2 * H + j]), o = sigmoidf_(g[3 * H + j]);
  const float c = f * c_prev[idx] + i * gg;
  const float h = o * tanhf(c);
  g[j] = i; g[H + j] = f; g[2 * H + j] = gg; g[3 * H + j] = o;
  c_out[idx] = c;
  h_out[idx] = h;
  if (h_bf) h_bf[idx] = __float2bfloat16_rn(h);
  if (hs) hs[(int64_t)m * hs_row + j] = h;
  if (hs_st) {
    if (st_is_bf16) reinterpret_cast<bf16*>(hs_st)[(int64_t)m * hs_row + j] = __float2bfloat16_rn(h);
    else reinterpret_cast<float*>(hs_st)[(int64_t)m * hs_row + j] = h;
  }
}
// backward of the cell: d h_t = dhs (caller, may be NULL) + carried ; writes d(pre-activations), updates d c in place
__global__ void seq_lstm_pw_bwd_kernel(const float* __restrict__ dhs, int64_t hs_row, const float* __restrict__ dh_carry, float* __restrict__ dc,
                                       const float* __restrict__ gates, const float* __restrict__ c_prev, const float* __restrict__ c_cur,
                                       float* __restrict__ dG, bf16* __restrict__ dG_bf, int M, int H) {
  pdl_wait();
  pdl_trigger();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * H) return;
  const int m = idx / H, j = idx % H;
  const float* g = gates + (int64_t)m * 4 * H;
  const float i = g[j], f = g[H + j], gg = g[2 * H + j], o = g[3 * H + j];
  const float tc = tanhf(c_cur[idx]);
  const float dh = (dhs ? dhs[(int64_t)m * hs_row + j] : 0.f) + dh_carry[idx];
  const float dct = dc[idx] + dh * o * (1.f - tc * tc);
  float v[4];
  v[0] = dct * gg * i * (1.f - i);
  v[1] = dct * c_prev[idx] * f * (1.f - f);
  v[2] = dct * i * (1.f - gg * gg);
  v[3] = dh * tc * o * (1.f - o);
  dc[idx] = dct * f;
#pragma unroll
  for (int q = 0; q < 4; q++) {
    dG[(int64_t)m * 4 * H + q * H + j] = v[q];
    if (dG_bf) dG_bf[(int64_t)m * 4 * H + q * H + j] = __float2bfloat16_rn(v[q]);
  }
}

static int seq_check(const lo_lstm_seq_args* a) {
  LO_CHECK_ARG(a != nullptr, "null args");
  LO_CHECK_ARG(a->S > 0 && a->M > 0 && a->I > 0 && a->H > 0, "S, M, I, H > 0");
  LO_CHECK_ARG(a->I % 8 == 0 && a->H % 8 == 0, "I, H multiples of 8");
  LO_CHECK_ARG(a->dt == LO_F32 || a->dt == LO_BF16, "dt");
  LO_CHECK_ARG(a->x && a->w_ih && a->w_hh && a->b_ih && a->b_hh && a->ws, "null pointer");
  LO_CHECK_ARG(a->x_row % 8 == 0 && a->x_step % 8 == 0, "x strides must be multiples of 8 elements");
  return LO_OK;
}

}  // namespace lo

using namespace lo;

extern "C" {

int64_t lo_sizeof_lstm_seq_args(void) { return (int64_t)sizeof(lo_lstm_seq_args); }

int64_t lo_lstm_seq_workspace_bytes(const lo_lstm_seq_args* a) {
  if (!a) return 0;
  lo_lstm_seq_args tmp = *a;
  tmp.ws = nullptr;
  return (int64_t)seq_carve(&tmp).bytes;
}

int lo_lstm_seq_forward(const lo_lstm_seq_args* a, void* stream) {
  LO_TRY(seq_check(a));
  LO_CHECK_ARG(a->hs || a->hs_st, "no output tensor");
  cudaStream_t st = (cudaStream_t)stream;
  const int S = a->S, M = a->M, I = a->I, H = a->H, G = 4 * a->H, dt = a->dt;
  const SeqWs w = seq_carve(a);
  const bool bf = dt == LO_BF16;
  const int impl = (a->impl == LO_IMPL_TC && bf) ? LO_IMPL_TC : LO_IMPL_SIMT;
  LO_DISPATCH_DT(dt, T, (seq_gather_kernel<T><<<LO_NUM_SMS * 8, 256, 0, st>>>((const T*)a->x, a->x_row, a->x_step, (T*)w.xt, S, M, I, a->reverse)));
  LO_LAUNCH_OK();
  seq_bias_sum_kernel<<<cdiv(G, 256), 256, 0, st>>>(a->b_ih, a->b_hh, w.bsum, G);
  LO_LAUNCH_OK();
  // hoisted input projection of every step
  LO_TRY(gemm_nt(w.xt, dt, I, a->w_ih, dt, I, w.gates, LO_F32, G, S * M, G, I, w.bsum, 0, 0, impl, st));
  seq_init_kernel<<<cdiv((long)M * H, 256), 256, 0, st>>>(a->h0, a->c0, w.h, w.c, w.h_bf, M * H);
  LO_LAUNCH_OK();
  for (int p = 0; p < S; p++) {
    const int t = a->reverse ? S - 1 - p : p;
    float* gp = w.gates + (int64_t)p * M * G;
    if (bf) LO_TRY(gemm_nt(w.h_bf + (int64_t)p * M * H, LO_BF16, H, a->w_hh, LO_BF16, H, gp, LO_F32, G, M, G, H, nullptr, 1, 0, impl, st));
    else LO_TRY(gemm_nt(w.h + (int64_t)p * M * H, LO_F32, H, a->w_hh, LO_F32, H, gp, LO_F32, G, M, G, H, nullptr, 1, 0, LO_IMPL_SIMT, st));
    const size_t es = bf ? 2 : 4;
    LO_CUDA(launch_pdl(seq_lstm_pw_fwd_kernel, dim3(cdiv((long)M * H, 256)), dim3(256), (size_t)0, st, gp,
                       (const float*)(w.c + (int64_t)p * M * H), w.c + (int64_t)(p + 1) * M * H, w.h + (int64_t)(p + 1) * M * H,
                       w.h_bf ? w.h_bf + (int64_t)(p + 1) * M * H : (bf16*)nullptr,
                       a->hs ? a->hs + (int64_t)t * a->hs_step : (float*)nullptr,
                       a->hs_st ? (void*)((char*)a->hs_st + (size_t)t * a->hs_step * es) : (void*)nullptr, bf ? 1 : 0, a->hs_row, M, H));
    LO_LAUNCH_OK();
  }
  return LO_OK;
}

int lo_lstm_seq_backward(const lo_lstm_seq_args* a, void* stream) {
  LO_TRY(seq_check(a));
  LO_CHECK_ARG(a->g_w_ih && a->g_w_hh && a->g_b_ih && a->g_b_hh, "null gradient buffer");
  cudaStream_t st = (cudaStream_t)stream;
  const int S = a->S, M = a->M, I = a->I, H = a->H, G = 4 * a->H, dt = a->dt;
  const SeqWs w = seq_carve(a);
  const bool bf = dt == LO_BF16;
  const int impl = (a->impl == LO_IMPL_TC && bf) ? LO_IMPL_TC : LO_IMPL_SIMT;
  // transposed weight copies for the d h / d x products (K-major operands)
  LO_DISPATCH_DT(dt, T, {
    transpose_kernel<T><<<dim3(cdiv(H, 32), cdiv(G, 32)), dim3(32, 8), 0, st>>>((const T*)a->w_hh, H, (T*)w.whhT, G, G, H);
    transpose_kernel<T><<<dim3(cdiv(I, 32), cdiv(G, 32)), dim3(32, 8), 0, st>>>((const T*)a->w_ih, I, (T*)w.wihT, G, G, I);
  });
  lo::g_launches += 1;
  LO_LAUNCH_OK();
  LO_CUDA(cudaMemsetAsync(w.dh, 0, (size_t)M * H * 4, st));
  LO_CUDA(cudaMemsetAsync(w.dc, 0, (size_t)M * H * 4, st));
  for (int p = S - 1; p >= 0; p--) {
    const int t = a->reverse ? S - 1 - p : p;
    float* dGp = w.dG + (int64_t)p * M * G;
    bf16* dGb = w.dG_bf ? w.dG_bf + (int64_t)p * M * G : nullptr;
    LO_CUDA(launch_pdl(seq_lstm_pw_bwd_kernel, dim3(cdiv((long)M * H, 256)), dim3(256), (size_t)0, st,
                       a->dhs ? a->dhs + (int64_t)t * a->hs_step : (const float*)nullptr, a->hs_row, (const float*)w.dh, w.dc,
                       (const float*)(w.gates + (int64_t)p * M * G), (const float*)(w.c + (int64_t)p * M * H),
                       (const float*)(w.c + (int64_t)(p + 1) * M * H), dGp, dGb, M, H));
    LO_LAUNCH_OK();
    // d h_{p-1} = d pre_p W_hh
    if (bf) LO_TRY(gemm_nt(dGb, LO_BF16, G, w.whhT, LO_BF16, G, w.dh, LO_F32, H, M, H, G, nullptr, 0, 0, impl, st));
    else LO_TRY(gemm_nt(dGp, LO_F32, G, w.whhT, LO_F32, G, w.dh, LO_F32, H, M, H, G, nullptr, 0, 0, LO_IMPL_SIMT, st));
  }
  if (a->dh0) LO_CUDA(cudaMemcpyAsync(a->dh0, w.dh, (size_t)M * H * 4, cudaMemcpyDeviceToDevice, st));
  if (a->dc0) LO_CUDA(cudaMemcpyAsync(a->dc0, w.dc, (size_t)M * H * 4, cudaMemcpyDeviceToDevice, st));
  // hoisted: weight gradients over the stacked steps, bias gradients, d x
  const void* dGs = bf ? (const void*)w.dG_bf : (const void*)w.dG;
  const void* hs_ = bf ? (const void*)w.h_bf : (const void*)w.h;       // slots 0..S-1 = h_{p-1}
  LO_TRY(gemm_tn(dGs, dt, G, hs_, dt, H, a->g_w_hh, LO_F32, H, G, H, S * M, 0, impl, st));
  LO_TRY(gemm_tn(dGs, dt, G, w.xt, dt, I, a->g_w_ih, LO_F32, I, G, I, S * M, 0, impl, st));
  LO_TRY(colsum(w.dG, LO_F32, a->g_b_ih, S * M, G, G, 0, st));
  LO_CUDA(cudaMemcpyAsync(a->g_b_hh, a->g_b_ih, (size_t)G * 4, cudaMemcpyDeviceToDevice, st));
  if (a->dx) {
    LO_TRY(gemm_nt(dGs, dt, G, w.wihT, dt, G, w.dxt, LO_F32, I, S * M, I, G, nullptr, 0, 0, impl, st));
    seq_scatter_kernel<<<LO_NUM_SMS * 8, 256, 0, st>>>(w.dxt, a->dx, a->dx_row, a->dx_step, S, M, I, a->reverse, a->dx_accumulate);
    LO_LAUNCH_OK();
  }
  return LO_OK;
}

}  // extern "C"
