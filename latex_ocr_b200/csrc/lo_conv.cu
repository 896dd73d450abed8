// Encoder kernels, CUDA-core versions (fp32 or bf16 storage, fp32 accumulate): the 6-conv "vanilla"
// stack of seq2seq_torch.py:31-57 in NHWC with [Cout][3][3][Cin] weights, its data/weight gradients,
// the max-pools and the timing-signal add.  The wgmma/TMA implicit-GEMM convolution is in lo_tc.cu.
#include "lo_common.cuh"

namespace lo {

// ------------------------------------------------------------------------------------------------
// conv1 (Cin = 1) + bias + ReLU + 2x2 max-pool, fused.  Memory-bound: 4 B/pixel in, 64 ch out.
// thread <-> (pooled position, group of 8 output channels)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ldpix(const float* p) { return *p; }
__device__ __forceinline__ float ldpix(const uint8_t* p) { return (float)*p; }

template <typename T, typename TI>
__global__ void __launch_bounds__(256) conv1_pool_fwd_kernel(const TI* __restrict__ img, const float* __restrict__ w,
                                                              const float* __restrict__ bias, T* __restrict__ out,
                                                              int N, int H, int W, float pscale, float poff,
                                                              uint8_t* __restrict__ code) {
  __shared__ float sw[64 * 9];
  __shared__ float sb[64];
  for (int i = threadIdx.x; i < 64 * 9; i += blockDim.x) sw[i] = w[i];
  if (threadIdx.x < 64) sb[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int Hp = H / 2, Wp = W / 2;
  const int64_t total = (int64_t)N * Hp * Wp * 8;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int cg = (int)(idx & 7);
    int64_t p = idx >> 3;
    const int wo = (int)(p % Wp); p /= Wp;
    const int ho = (int)(p % Hp);
    const int n = (int)(p / Hp);
    float x[4][4];
    const TI* ib = img + (int64_t)n * H * W;
#pragma unroll
    for (int dy = 0; dy < 4; dy++) {
      const int hi = 2 * ho - 1 + dy;
#pragma unroll
      for (int dx = 0; dx < 4; dx++) {
        const int wi = 2 * wo - 1 + dx;
        x[dy][dx] = (hi >= 0 && hi < H && wi >= 0 && wi < W) ? fmaf(ldpix(ib + (int64_t)hi * W + wi), pscale, poff) : 0.f;
      }
    }
    float o[8];
    uint32_t cw[2] = {0u, 0u};
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const float* wc = sw + (cg * 8 + c) * 9;
      float best = -INFINITY;
      uint32_t bi = 0;
#pragma unroll
      for (int py = 0; py < 2; py++)
#pragma unroll
        for (int px = 0; px < 2; px++) {
          float s = sb[cg * 8 + c];
#pragma unroll
          for (int r = 0; r < 3; r++)
#pragma unroll
            for (int q = 0; q < 3; q++) s = fmaf(wc[r * 3 + q], x[py + r][px + q], s);
          if (s > best) { best = s; bi = py * 2 + px; }        // first maximum in scan order (PyTorch max_pool2d)
        }
      o[c] = fmaxf(best, 0.f);
      // training: window index of the pool arg-max (bits 0-1) and the ReLU bit (bit 2) for the weight-gradient kernel
      cw[c >> 2] |= (bi | (best > 0.f ? 4u : 0u)) << (8 * (c & 3));
    }
    const int64_t o_off = (((int64_t)n * Hp + ho) * Wp + wo) * 64 + cg * 8;
    st8(out + o_off, o);
    if (code) *reinterpret_cast<uint2*>(code + o_off) = make_uint2(cw[0], cw[1]);
  }
}

// conv1 weight / bias gradient: every block adds its partial sums (64 channels x (9 taps + bias)) onto the zeroed dw / db with fp32
// atomics.  Option "deterministic": it stores them in its own slot of g_conv1_part instead and conv1_wgrad_reduce_kernel adds the
// slots in block order; the slots are a device buffer of the library, so with that option two conv1 weight-gradient calls must not
// run concurrently on one device.
constexpr int C1_PART = 64 * 10;
constexpr int C1_MAXBLOCKS = LO_NUM_SMS * 4;
__device__ float g_conv1_part[C1_MAXBLOCKS][C1_PART];

__device__ __forceinline__ void conv1_wgrad_block_partial(const float (&gw)[8][9], const float (&gb)[8], int cg, int lane, float* dw,
                                                          float* db, int ordered) {
  float* part = g_conv1_part[blockIdx.x];
#pragma unroll
  for (int c = 0; c < 8; c++) {
    const float s = warp_sum(gb[c]);
    if (lane == 0) {
      if (ordered) part[(cg * 8 + c) * 10 + 9] = s;
      else atomicAdd(db + cg * 8 + c, s);
    }
#pragma unroll
    for (int k = 0; k < 9; k++) {
      const float t = warp_sum(gw[c][k]);
      if (lane == 0) {
        if (ordered) part[(cg * 8 + c) * 10 + k] = t;
        else atomicAdd(dw + (cg * 8 + c) * 9 + k, t);
      }
    }
  }
}

__global__ void conv1_wgrad_reduce_kernel(float* __restrict__ dw, float* __restrict__ db, int nblocks) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C1_PART) return;
  float s = 0.f;
  for (int b = 0; b < nblocks; b++) s += g_conv1_part[b][i];
  const int c = i / 10, k = i % 10;
  if (k == 9) db[c] = s;
  else dw[c * 9 + k] = s;
}

// Decodes one arg-max / ReLU code byte of conv1_pool_fwd_kernel: returns the gradient of the winning conv position (g, or 0 when
// the ReLU bit is clear: relu'(0) = 0) and its window position (py, px).  The weight and the data gradient both decode through
// this, so they agree on the arg-max and on relu'(0).
__device__ __forceinline__ float conv1_code_decode(uint32_t cd, float g, bool& py, bool& px) {
  px = cd & 1u;
  py = cd & 2u;
  return (cd & 4u) ? g : 0.f;
}

// conv1 weight gradient from the arg-max / ReLU codes the forward kernel saved: no recomputation of conv1 (36 of the 84 FMA slots
// per pooled output and channel), the 3x3 window of the winning position is selected with 21 selects instead of 27 masked FMAs.
// warp <-> 8 channels, lane <-> pooled position (as conv1_pool_wgrad_kernel below).
template <typename T, typename TI>
__global__ void __launch_bounds__(256) conv1_pool_wgrad_code_kernel(const TI* __restrict__ img, const uint8_t* __restrict__ code,
                                                                     const T* __restrict__ dpool, float* __restrict__ dw,
                                                                     float* __restrict__ db, int N, int H, int W, float pscale,
                                                                     float poff, int ordered) {
  const int Hp = H / 2, Wp = W / 2;
  const int lane = threadIdx.x & 31, cg = threadIdx.x >> 5;
  const int64_t npos = (int64_t)N * Hp * Wp;
  float gw[8][9];
  float gb[8];
#pragma unroll
  for (int c = 0; c < 8; c++) {
    gb[c] = 0.f;
#pragma unroll
    for (int k = 0; k < 9; k++) gw[c][k] = 0.f;
  }
  for (int64_t p0 = (int64_t)blockIdx.x * 32; p0 < npos; p0 += (int64_t)gridDim.x * 32) {
    const int64_t pp = p0 + lane;
    if (pp >= npos) continue;
    int64_t p = pp;
    const int wo = (int)(p % Wp); p /= Wp;
    const int ho = (int)(p % Hp);
    const int n = (int)(p / Hp);
    float x[4][4];
    const TI* ib = img + (int64_t)n * H * W;
#pragma unroll
    for (int dy = 0; dy < 4; dy++) {
      const int hi = 2 * ho - 1 + dy;
#pragma unroll
      for (int dx = 0; dx < 4; dx++) {
        const int wi = 2 * wo - 1 + dx;
        x[dy][dx] = (hi >= 0 && hi < H && wi >= 0 && wi < W) ? fmaf(ldpix(ib + (int64_t)hi * W + wi), pscale, poff) : 0.f;
      }
    }
    float g[8];
    ld8(dpool + pp * 64 + cg * 8, g);
    const uint2 cw2 = *reinterpret_cast<const uint2*>(code + pp * 64 + cg * 8);
    const uint32_t cw[2] = {cw2.x, cw2.y};
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const uint32_t cd = (cw[c >> 2] >> (8 * (c & 3))) & 0xffu;
      bool py, px;
      const float gg = conv1_code_decode(cd, g[c], py, px);
      gb[c] += gg;
      float xc[4][3];
#pragma unroll
      for (int dy = 0; dy < 4; dy++)
#pragma unroll
        for (int q = 0; q < 3; q++) xc[dy][q] = px ? x[dy][q + 1] : x[dy][q];
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int q = 0; q < 3; q++) gw[c][r * 3 + q] = fmaf(gg, py ? xc[r + 1][q] : xc[r][q], gw[c][r * 3 + q]);
    }
  }
  conv1_wgrad_block_partial(gw, gb, cg, lane, dw, db, ordered);
}

// conv1 data gradient through its ReLU and 2x2 max-pool, from the same codes:
//   dimg[n,y,x] = scale * sum_{r,q} sum_c w[c][r][q] * dpre[n, y+1-r, x+1-q, c]
// with dpre = dpool at the winning conv position of each pooled output (0 elsewhere, and 0 where the ReLU bit is clear).
// A block owns C1D_TH x C1D_TW pooled positions of one image and computes them plus a ring of one position (C1D_EH x C1D_EW,
// two per thread; the ring is computed again by the neighbouring block).  A thread sums the 64 channels of its pooled position,
// in channel order, into the 4x4 pixel patch their winning conv positions touch: 9 products per channel, placed by selects on
// the window position.  The patches go to shared memory; each owned pixel then adds the (up to) four patches that cover it in a
// fixed order and is written by that one thread.  No atomics: the result is bit-reproducible.
constexpr int C1D_EH = 16, C1D_EW = 32, C1D_TH = C1D_EH - 2, C1D_TW = C1D_EW - 2;
constexpr int C1D_PS = 17;                // patch stride in shared memory (16 + 1: neighbouring patches fall in different banks)

template <typename T>
__global__ void __launch_bounds__(256) conv1_pool_dgrad_code_kernel(const uint8_t* __restrict__ code, const T* __restrict__ dpool,
                                                                     const float* __restrict__ w, float scale,
                                                                     float* __restrict__ dimg, int H, int W) {
  __shared__ float sw[64 * 9];
  __shared__ float patch[C1D_EH * C1D_EW * C1D_PS];
  for (int i = threadIdx.x; i < 64 * 9; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int Hp = H / 2, Wp = W / 2;
  const int n = blockIdx.z;
  const int h0 = blockIdx.y * C1D_TH, w0 = blockIdx.x * C1D_TW;     // first owned pooled position
  for (int e = threadIdx.x; e < C1D_EH * C1D_EW; e += blockDim.x) {
    const int ho = h0 - 1 + e / C1D_EW, wo = w0 - 1 + e % C1D_EW;
    if (ho < 0 || ho >= Hp || wo < 0 || wo >= Wp) continue;        // outside the image: never read below
    const int64_t pp = (((int64_t)n * Hp + ho) * Wp + wo) * 64;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 16; i++) acc[i >> 2][i & 3] = 0.f;
#pragma unroll 1
    for (int cg = 0; cg < 8; cg++) {
      float g[8];
      ld8(dpool + pp + cg * 8, g);
      const uint2 cw2 = *reinterpret_cast<const uint2*>(code + pp + cg * 8);
      const uint32_t cw[2] = {cw2.x, cw2.y};
#pragma unroll
      for (int c = 0; c < 8; c++) {
        bool py, px;
        const float gg = conv1_code_decode((cw[c >> 2] >> (8 * (c & 3))) & 0xffu, g[c], py, px);
        const float* wc = sw + (cg * 8 + c) * 9;
        float u[3][4];                    // row r of the tap products, shifted right by px
#pragma unroll
        for (int r = 0; r < 3; r++) {
          const float t0 = gg * wc[r * 3], t1 = gg * wc[r * 3 + 1], t2 = gg * wc[r * 3 + 2];
          u[r][0] = px ? 0.f : t0;
          u[r][1] = px ? t0 : t1;
          u[r][2] = px ? t1 : t2;
          u[r][3] = px ? t2 : 0.f;
        }
#pragma unroll
        for (int dx = 0; dx < 4; dx++) {  // ... and down by py
          acc[0][dx] += py ? 0.f : u[0][dx];
          acc[1][dx] += py ? u[0][dx] : u[1][dx];
          acc[2][dx] += py ? u[1][dx] : u[2][dx];
          acc[3][dx] += py ? u[2][dx] : 0.f;
        }
      }
    }
    float* ps = patch + e * C1D_PS;       // patch pixel (dy, dx) is image pixel (2ho-1+dy, 2wo-1+dx)
#pragma unroll
    for (int i = 0; i < 16; i++) ps[i] = acc[i >> 2][i & 3];
  }
  __syncthreads();
  // owned pixels: the 2x2 blocks under the owned pooled positions; the last tile row / column also owns the image row / column an
  // odd H / W leaves outside every pool window (it receives taps of the conv row / column before it, but no gradient of its own)
  const int y0 = 2 * h0, x0 = 2 * w0;
  const int y1 = (h0 + C1D_TH >= Hp) ? H : 2 * (h0 + C1D_TH), x1 = (w0 + C1D_TW >= Wp) ? W : 2 * (w0 + C1D_TW);
  const int tw = x1 - x0, npix = (y1 - y0) * tw;
  for (int i = threadIdx.x; i < npix; i += blockDim.x) {
    const int y = y0 + i / tw, x = x0 + i % tw;
    float s = 0.f;
#pragma unroll
    for (int a = 0; a < 2; a++) {
      const int ho = ((y + 1) >> 1) - 1 + a;                       // the two pooled rows whose patches (rows 2ho-1..2ho+2) hold y
      if (ho < 0 || ho >= Hp) continue;
#pragma unroll
      for (int b = 0; b < 2; b++) {
        const int wo = ((x + 1) >> 1) - 1 + b;
        if (wo < 0 || wo >= Wp) continue;
        s += patch[((ho - h0 + 1) * C1D_EW + (wo - w0 + 1)) * C1D_PS + (y - 2 * ho + 1) * 4 + (x - 2 * wo + 1)];
      }
    }
    dimg[((int64_t)n * H + y) * W + x] = s * scale;
  }
}

// conv1 weight gradient from the pooled-output gradient (recompute conv1 -> argmax + ReLU mask).
// warp <-> 8 channels (blockDim = 256: warp id = channel group), lane <-> pooled position.
template <typename T, typename TI>
__global__ void __launch_bounds__(256) conv1_pool_wgrad_kernel(const TI* __restrict__ img, const float* __restrict__ w,
                                                                const float* __restrict__ bias, const T* __restrict__ dpool,
                                                                float* __restrict__ dw, float* __restrict__ db,
                                                                int N, int H, int W, float pscale, float poff, int ordered) {
  __shared__ float sw[64 * 9];
  __shared__ float sb[64];
  for (int i = threadIdx.x; i < 64 * 9; i += blockDim.x) sw[i] = w[i];
  if (threadIdx.x < 64) sb[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int Hp = H / 2, Wp = W / 2;
  const int lane = threadIdx.x & 31, cg = threadIdx.x >> 5;
  const int64_t npos = (int64_t)N * Hp * Wp;
  float gw[8][9];
  float gb[8];
#pragma unroll
  for (int c = 0; c < 8; c++) {
    gb[c] = 0.f;
#pragma unroll
    for (int k = 0; k < 9; k++) gw[c][k] = 0.f;
  }
  for (int64_t p0 = (int64_t)blockIdx.x * 32; p0 < npos; p0 += (int64_t)gridDim.x * 32) {
    const int64_t pp = p0 + lane;
    if (pp >= npos) continue;
    int64_t p = pp;
    const int wo = (int)(p % Wp); p /= Wp;
    const int ho = (int)(p % Hp);
    const int n = (int)(p / Hp);
    float x[4][4];
    const TI* ib = img + (int64_t)n * H * W;
#pragma unroll
    for (int dy = 0; dy < 4; dy++) {
      const int hi = 2 * ho - 1 + dy;
#pragma unroll
      for (int dx = 0; dx < 4; dx++) {
        const int wi = 2 * wo - 1 + dx;
        x[dy][dx] = (hi >= 0 && hi < H && wi >= 0 && wi < W) ? fmaf(ldpix(ib + (int64_t)hi * W + wi), pscale, poff) : 0.f;
      }
    }
    float g[8];
    ld8(dpool + pp * 64 + cg * 8, g);
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const float* wc = sw + (cg * 8 + c) * 9;
      float best = -INFINITY;
      int bi = 0;
#pragma unroll
      for (int py = 0; py < 2; py++)
#pragma unroll
        for (int px = 0; px < 2; px++) {
          float s = sb[cg * 8 + c];
#pragma unroll
          for (int r = 0; r < 3; r++)
#pragma unroll
            for (int q = 0; q < 3; q++) s = fmaf(wc[r * 3 + q], x[py + r][px + q], s);
          if (s > best) { best = s; bi = py * 2 + px; }   // first maximum in scan order (PyTorch max_pool2d)
        }
      const float gg = (best > 0.f) ? g[c] : 0.f;
      gb[c] += gg;
#pragma unroll
      for (int py = 0; py < 2; py++)
#pragma unroll
        for (int px = 0; px < 2; px++) {
          const float sel = (bi == py * 2 + px) ? gg : 0.f;
#pragma unroll
          for (int r = 0; r < 3; r++)
#pragma unroll
            for (int q = 0; q < 3; q++) gw[c][r * 3 + q] = fmaf(sel, x[py + r][px + q], gw[c][r * 3 + q]);
        }
    }
  }
  conv1_wgrad_block_partial(gw, gb, cg, lane, dw, db, ordered);
}

// ------------------------------------------------------------------------------------------------
// implicit-GEMM 3x3 convolution, CUDA cores: M = N*Ho*Wo, Ngemm = Cout, K = 9*Cin (tap-major).
// 64x64x16 tile, 256 threads, 4x4 micro-tile.  Cin % 16 == 0 so a K chunk never straddles a tap.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) conv3x3_igemm_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                             const float* __restrict__ bias, const T* __restrict__ mask,
                                                             T* __restrict__ y, int N, int H, int W, int Cin, int Cout,
                                                             int pad, int relu) {
  constexpr int BM = 64, BN = 64, BK = 16;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int Ho = H + 2 * pad - 2, Wo = W + 2 * pad - 2;
  const int64_t Mtot = (int64_t)N * Ho * Wo;
  const int K = 9 * Cin;
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;
  const int64_t m0 = (int64_t)blockIdx.x * BM;     // M tiles on grid.x (up to 2^31 - 1 of them; grid.y stops at 65535)
  const int n0 = blockIdx.y * BN;
  // this thread loads A rows (tid/16 + 16*j), k = tid%16
  const int lk = tid % BK;
  int a_h[4], a_w[4];
  int64_t a_img[4];
  bool a_ok[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int64_t m = m0 + tid / BK + 16 * j;
    a_ok[j] = m < Mtot;
    int64_t p = a_ok[j] ? m : 0;
    a_w[j] = (int)(p % Wo); p /= Wo;
    a_h[j] = (int)(p % Ho);
    a_img[j] = (p / Ho) * (int64_t)H * W;
  }
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += BK) {
    const int tap = k0 / Cin, ci0 = k0 % Cin;
    const int r = tap / 3 - pad, s = tap % 3 - pad;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int hi = a_h[j] + r, wi = a_w[j] + s;
      float v = 0.f;
      if (a_ok[j] && hi >= 0 && hi < H && wi >= 0 && wi < W)
        v = ldf(x + (a_img[j] + (int64_t)hi * W + wi) * Cin + ci0 + lk);
      As[lk][tid / BK + 16 * j] = v;
    }
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int n = tid / BK + 16 * j;
      float v = 0.f;
      if (n0 + n < Cout) v = ldf(w + (int64_t)(n0 + n) * K + k0 + lk);
      Bs[lk][n] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; k++) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= Mtot) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int n = n0 + tx * 4 + j;
      if (n >= Cout) continue;
      float v = acc[i][j];
      if (bias) v += bias[n];
      if (relu) v = fmaxf(v, 0.f);
      if (mask && !(ldf(mask + m * Cout + n) > 0.f)) v = 0.f;
      stf(y + m * Cout + n, v);
    }
  }
}

// weight gradient: dw[co][tap][ci] += sum_{positions in split} dy[pos][co] * x[pos+tap][ci]
// grid: (Cin/64, Cout/64, 9*splits)
template <typename T>
__global__ void __launch_bounds__(256) conv3x3_wgrad_kernel(const T* __restrict__ x, const T* __restrict__ dy,
                                                             float* __restrict__ dw, int N, int H, int W, int Cin, int Cout,
                                                             int pad, int splits) {
  constexpr int BM = 64, BN = 64, BK = 16;
  __shared__ __align__(16) float As[BK][BM + 4];   // dy^T : [pos][co]
  __shared__ __align__(16) float Bs[BK][BN + 4];   // x    : [pos][ci]
  const int Ho = H + 2 * pad - 2, Wo = W + 2 * pad - 2;
  const int64_t P = (int64_t)N * Ho * Wo;
  const int tap = blockIdx.z / splits, sp = blockIdx.z % splits;
  const int r = tap / 3 - pad, s = tap % 3 - pad;
  const int64_t per = ((P + splits - 1) / splits + BK - 1) / BK * BK;
  const int64_t pbeg = sp * per, pend = min(P, pbeg + per);
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int co0 = blockIdx.y * BM, ci0 = blockIdx.x * BN;
  const int lc = tid % 64;      // channel within tile (fast index)
  const int lp = tid / 64;      // position lane 0..3 ; loads positions lp + 4*j
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
  for (int64_t p0 = pbeg; p0 < pend; p0 += BK) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int kk = lp + 4 * j;
      const int64_t pos = p0 + kk;
      float va = 0.f, vb = 0.f;
      if (pos < pend) {
        if (co0 + lc < Cout) va = ldf(dy + pos * Cout + co0 + lc);
        int64_t q = pos;
        const int wo = (int)(q % Wo); q /= Wo;
        const int ho = (int)(q % Ho);
        const int64_t n = q / Ho;
        const int hi = ho + r, wi = wo + s;
        if (hi >= 0 && hi < H && wi >= 0 && wi < W && ci0 + lc < Cin)
          vb = ldf(x + ((n * H + hi) * W + wi) * Cin + ci0 + lc);
      }
      As[kk][lc] = va;
      Bs[kk][lc] = vb;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; k++) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int co = co0 + ty * 4 + i;
    if (co >= Cout) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int ci = ci0 + tx * 4 + j;
      if (ci >= Cin) continue;
      atomicAdd(dw + ((int64_t)co * 9 + tap) * Cin + ci, acc[i][j]);
    }
  }
}

template <typename T>
__global__ void weight_flip_kernel(const T* __restrict__ w, T* __restrict__ wt, int Cin, int Cout) {
  const int64_t total = (int64_t)Cin * 9 * Cout;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int co = (int)(i % Cout);
    int64_t q = i / Cout;
    const int tap = (int)(q % 9);
    const int ci = (int)(q / 9);
    wt[i] = w[((int64_t)co * 9 + (8 - tap)) * Cin + ci];
  }
}

template <typename T>
__global__ void maxpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int N, int H, int W, int C, int kh, int kw) {
  const int Ho = H / kh, Wo = W / kw, C8 = C / 8;
  const int64_t total = (int64_t)N * Ho * Wo * C8;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % C8);
    int64_t p = idx / C8;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int64_t n = p / Ho;
    float best[8];
#pragma unroll
    for (int c = 0; c < 8; c++) best[c] = -INFINITY;
    for (int a = 0; a < kh; a++)
      for (int b = 0; b < kw; b++) {
        float v[8];
        ld8(x + ((n * H + ho * kh + a) * W + wo * kw + b) * C + c8 * 8, v);
#pragma unroll
        for (int c = 0; c < 8; c++) best[c] = fmaxf(best[c], v[c]);
      }
    st8(y + ((n * Ho + ho) * Wo + wo) * C + c8 * 8, best);
  }
}

// dx over the pooled region (rows < Ho*kh, cols < Wo*kw); leftover rows/cols are zeroed by the launcher.
template <typename T>
__global__ void maxpool_bwd_kernel(const T* __restrict__ x, const T* __restrict__ dy, T* __restrict__ dx,
                                   int N, int H, int W, int C, int kh, int kw) {
  const int Ho = H / kh, Wo = W / kw, C8 = C / 8;
  const int64_t total = (int64_t)N * Ho * Wo * C8;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % C8);
    int64_t p = idx / C8;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int64_t n = p / Ho;
    float g[8], best[8];
    int bi[8];
    ld8(dy + ((n * Ho + ho) * Wo + wo) * C + c8 * 8, g);
#pragma unroll
    for (int c = 0; c < 8; c++) { best[c] = -INFINITY; bi[c] = 0; }
    for (int a = 0; a < kh; a++)
      for (int b = 0; b < kw; b++) {
        float v[8];
        ld8(x + ((n * H + ho * kh + a) * W + wo * kw + b) * C + c8 * 8, v);
#pragma unroll
        for (int c = 0; c < 8; c++)
          if (v[c] > best[c]) { best[c] = v[c]; bi[c] = a * kw + b; }
      }
    for (int a = 0; a < kh; a++)
      for (int b = 0; b < kw; b++) {
        float o[8];
#pragma unroll
        for (int c = 0; c < 8; c++) o[c] = (bi[c] == a * kw + b && best[c] > 0.f) ? g[c] : 0.f;
        st8(dx + ((n * H + ho * kh + a) * W + wo * kw + b) * C + c8 * 8, o);
      }
  }
}

template <typename T>
__global__ void add_table_kernel(const T* __restrict__ y, const float* __restrict__ table, T* __restrict__ out,
                                 int64_t total8, int64_t hwc8) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total8; i += (int64_t)gridDim.x * blockDim.x) {
    float v[8], t[8];
    ld8(y + i * 8, v);
    ld8(table + (i % hwc8) * 8, t);
#pragma unroll
    for (int c = 0; c < 8; c++) v[c] += t[c];
    st8(out + i * 8, v);
  }
}

template <typename T>
__global__ void relu_mask_cast_kernel(const float* __restrict__ g, const T* __restrict__ y, T* __restrict__ out, int64_t n8) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    float a[8], b[8];
    ld8(g + i * 8, a);
    ld8(y + i * 8, b);
#pragma unroll
    for (int c = 0; c < 8; c++) a[c] = b[c] > 0.f ? a[c] : 0.f;
    st8(out + i * 8, a);
  }
}

static inline int grid_for(int64_t work, int threads) {
  int64_t b = (work + threads - 1) / threads;
  const int64_t cap = LO_NUM_SMS * 16;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}


// ------------------------------------------------------------------------------------------------
// General strided convolution as im2col + GEMM: the 'cnn' encoder variant's Conv2d(512, 512, (2,4), stride 2, padding 1)
// (seq2seq_torch.py:80).  col [N*Ho*Wo][R*S*C] (tap-major like the 3x3 kernels' K order), 8 channels per thread.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void im2col_kernel(const T* __restrict__ x, T* __restrict__ col, int N, int H, int W, int C, int R, int S, int stride,
                              int pad, int Ho, int Wo) {
  const int C8 = C / 8;
  const int64_t total = (int64_t)N * Ho * Wo * R * S * C8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % C8);
    int64_t q = i / C8;
    const int s = (int)(q % S); q /= S;
    const int r = (int)(q % R); q /= R;
    const int wo = (int)(q % Wo); q /= Wo;
    const int ho = (int)(q % Ho);
    const int n = (int)(q / Ho);
    const int hi = ho * stride - pad + r, wi = wo * stride - pad + s;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (hi >= 0 && hi < H && wi >= 0 && wi < W) ld8(x + (((int64_t)n * H + hi) * W + wi) * C + c8 * 8, v);
    st8(col + i * 8, v);
  }
}
// dx[n][hi][wi][c] = sum over the windows (ho,r), (wo,s) that cover (hi,wi) of dcol[n][ho][wo][r][s][c]  [* (mask > 0)]  — a gather
template <typename T>
__global__ void col2im_kernel(const T* __restrict__ dcol, const T* __restrict__ mask, T* __restrict__ dx, int N, int H, int W, int C,
                              int R, int S, int stride, int pad, int Ho, int Wo) {
  const int C8 = C / 8;
  const int64_t total = (int64_t)N * H * W * C8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % C8);
    int64_t q = i / C8;
    const int wi = (int)(q % W); q /= W;
    const int hi = (int)(q % H);
    const int n = (int)(q / H);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int r = 0; r < R; r++) {
      const int hn = hi + pad - r;
      if (hn < 0 || hn % stride) continue;
      const int ho = hn / stride;
      if (ho >= Ho) continue;
      for (int s2 = 0; s2 < S; s2++) {
        const int wn = wi + pad - s2;
        if (wn < 0 || wn % stride) continue;
        const int wo = wn / stride;
        if (wo >= Wo) continue;
        float v[8];
        ld8(dcol + (((((int64_t)n * Ho + ho) * Wo + wo) * R + r) * S + s2) * C + c8 * 8, v);
#pragma unroll
        for (int k = 0; k < 8; k++) acc[k] += v[k];
      }
    }
    if (mask) {
      float m[8];
      ld8(mask + i * 8, m);
#pragma unroll
      for (int k = 0; k < 8; k++) acc[k] = m[k] > 0.f ? acc[k] : 0.f;
    }
    st8(dx + i * 8, acc);
  }
}
// out[n][k] = in[k][n]
template <typename T>
__global__ void transpose2d_kernel(const T* __restrict__ in, int64_t ld_in, T* __restrict__ out, int64_t ld_out, int K, int Nn) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += 8)
    if (k0 + i < K && n0 + threadIdx.x < Nn) tile[i][threadIdx.x] = ldf(in + (int64_t)(k0 + i) * ld_in + n0 + threadIdx.x);
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8)
    if (n0 + i < Nn && k0 + threadIdx.x < K) stf(out + (int64_t)(n0 + i) * ld_out + k0 + threadIdx.x, tile[threadIdx.x][i]);
}

}  // namespace lo

using namespace lo;

extern "C" {

static int conv1_fwd(const void* img, int u8, const float* w, const float* bias, void* out, int dt, int N, int H, int W, cudaStream_t st,
                     float pscale = 1.f, float poff = 0.f, uint8_t* code = nullptr) {
  LO_CHECK_ARG(img && w && bias && out, "null pointer");
  LO_CHECK_ARG(N > 0 && H >= 2 && W >= 2, "shape");
  const int64_t work = (int64_t)N * (H / 2) * (W / 2) * 8;
  const int grid = grid_for(work, 256);
  if (u8) {
    LO_DISPATCH_DT(dt, T, (conv1_pool_fwd_kernel<T, uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)img, w, bias, (T*)out, N, H, W, pscale, poff, code)));
  } else {
    LO_DISPATCH_DT(dt, T, (conv1_pool_fwd_kernel<T, float><<<grid, 256, 0, st>>>((const float*)img, w, bias, (T*)out, N, H, W, pscale, poff, code)));
  }
  LO_LAUNCH_OK();
  return LO_OK;
}

static int conv1_wgrad(const void* img, int u8, const float* w, const float* bias, const void* dpool, int dt, float* dw, float* db,
                       int N, int H, int W, cudaStream_t st, float pscale = 1.f, float poff = 0.f, const uint8_t* code = nullptr) {
  LO_CHECK_ARG(img && w && bias && dpool && dw && db, "null pointer");
  const int ordered = g_opt_det;
  if (!ordered) {
    LO_CUDA(cudaMemsetAsync(dw, 0, 64 * 9 * sizeof(float), st));
    LO_CUDA(cudaMemsetAsync(db, 0, 64 * sizeof(float), st));
  }
  const int64_t npos = (int64_t)N * (H / 2) * (W / 2);
  int grid = (int)((npos + 31) / 32);
  if (grid > C1_MAXBLOCKS) grid = C1_MAXBLOCKS;
  if (code) {
    if (u8) {
      LO_DISPATCH_DT(dt, T, (conv1_pool_wgrad_code_kernel<T, uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)img, code, (const T*)dpool, dw, db, N, H, W, pscale, poff, ordered)));
    } else {
      LO_DISPATCH_DT(dt, T, (conv1_pool_wgrad_code_kernel<T, float><<<grid, 256, 0, st>>>((const float*)img, code, (const T*)dpool, dw, db, N, H, W, pscale, poff, ordered)));
    }
    LO_LAUNCH_OK();
  } else if (u8) {
    LO_DISPATCH_DT(dt, T, (conv1_pool_wgrad_kernel<T, uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)img, w, bias, (const T*)dpool, dw, db, N, H, W, pscale, poff, ordered)));
    LO_LAUNCH_OK();
  } else {
    LO_DISPATCH_DT(dt, T, (conv1_pool_wgrad_kernel<T, float><<<grid, 256, 0, st>>>((const float*)img, w, bias, (const T*)dpool, dw, db, N, H, W, pscale, poff, ordered)));
    LO_LAUNCH_OK();
  }
  if (ordered) {
    conv1_wgrad_reduce_kernel<<<cdiv(C1_PART, 128), 128, 0, st>>>(dw, db, grid);
    LO_LAUNCH_OK();
  }
  return LO_OK;
}

int lo_conv1_pool_forward(const float* img, const float* w, const float* bias, void* out, int dt, int N, int H, int W,
                          void* stream) {
  return conv1_fwd(img, 0, w, bias, out, dt, N, H, W, (cudaStream_t)stream);
}
int lo_conv1_pool_forward_u8(const uint8_t* img, const float* w, const float* bias, void* out, int dt, int N, int H, int W,
                             void* stream) {
  return conv1_fwd(img, 1, w, bias, out, dt, N, H, W, (cudaStream_t)stream);
}
int lo_conv1_pool_wgrad(const float* img, const float* w, const float* bias, const void* dpool, int dt, float* dw,
                        float* db, int N, int H, int W, void* stream) {
  return conv1_wgrad(img, 0, w, bias, dpool, dt, dw, db, N, H, W, (cudaStream_t)stream);
}
int lo_conv1_pool_wgrad_u8(const uint8_t* img, const float* w, const float* bias, const void* dpool, int dt, float* dw,
                           float* db, int N, int H, int W, void* stream) {
  return conv1_wgrad(img, 1, w, bias, dpool, dt, dw, db, N, H, W, (cudaStream_t)stream);
}

int lo_conv1_pool_forward_norm(const void* img, int img_is_u8, float scale, float offset, const float* w, const float* bias, void* out,
                               int dt, int N, int H, int W, void* stream) {
  return conv1_fwd(img, img_is_u8, w, bias, out, dt, N, H, W, (cudaStream_t)stream, scale, offset);
}
int lo_conv1_pool_forward_code(const void* img, int img_is_u8, float scale, float offset, const float* w, const float* bias, void* out,
                               uint8_t* code, int dt, int N, int H, int W, void* stream) {
  return conv1_fwd(img, img_is_u8, w, bias, out, dt, N, H, W, (cudaStream_t)stream, scale, offset, code);
}
int lo_conv1_pool_wgrad_code(const void* img, int img_is_u8, float scale, float offset, const uint8_t* code, const void* dpool, int dt,
                             float* dw, float* db, int N, int H, int W, void* stream) {
  LO_CHECK_ARG(code, "null code");
  static const float dummy[1] = {0.f};
  return conv1_wgrad(img, img_is_u8, dummy, dummy, dpool, dt, dw, db, N, H, W, (cudaStream_t)stream, scale, offset, code);
}
int lo_conv1_pool_wgrad_norm(const void* img, int img_is_u8, float scale, float offset, const float* w, const float* bias,
                             const void* dpool, int dt, float* dw, float* db, int N, int H, int W, void* stream) {
  return conv1_wgrad(img, img_is_u8, w, bias, dpool, dt, dw, db, N, H, W, (cudaStream_t)stream, scale, offset);
}
int lo_conv1_pool_dgrad_code(const uint8_t* code, const void* dpool, int dt, const float* w, float scale, float* dimg, int N, int H,
                             int W, void* stream) {
  LO_CHECK_ARG(code && dpool && w && dimg, "null pointer");
  LO_CHECK_ARG(dt == LO_F32 || dt == LO_BF16, "dt must be LO_F32 or LO_BF16");
  LO_CHECK_ARG(N >= 1 && H >= 2 && W >= 2, "shape (N >= 1, H >= 2, W >= 2)");
  LO_CHECK_ARG(N <= 65535 && (H / 2 + C1D_TH - 1) / C1D_TH <= 65535, "shape (N or H too large for the grid)");
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(cdiv(W / 2, C1D_TW), cdiv(H / 2, C1D_TH), N);
  LO_DISPATCH_DT(dt, T, (conv1_pool_dgrad_code_kernel<T><<<grid, 256, 0, st>>>(code, (const T*)dpool, w, scale, dimg, H, W)));
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_im2col(const void* x, void* col, int dt, int N, int H, int W, int C, int R, int S, int stride, int pad, void* stream) {
  LO_CHECK_ARG(x && col && N > 0 && C % 8 == 0 && R > 0 && S > 0 && stride > 0 && pad >= 0, "null pointer / shape (C%8)");
  const int Ho = (H + 2 * pad - R) / stride + 1, Wo = (W + 2 * pad - S) / stride + 1;
  LO_CHECK_ARG(Ho > 0 && Wo > 0, "empty output");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t work = (int64_t)N * Ho * Wo * R * S * (C / 8);
  LO_DISPATCH_DT(dt, T, (im2col_kernel<T><<<grid_for(work, 256), 256, 0, st>>>((const T*)x, (T*)col, N, H, W, C, R, S, stride, pad, Ho, Wo)));
  LO_LAUNCH_OK();
  return LO_OK;
}
int lo_col2im(const void* dcol, const void* mask, void* dx, int dt, int N, int H, int W, int C, int R, int S, int stride, int pad,
              void* stream) {
  LO_CHECK_ARG(dcol && dx && N > 0 && C % 8 == 0 && R > 0 && S > 0 && stride > 0 && pad >= 0, "null pointer / shape (C%8)");
  const int Ho = (H + 2 * pad - R) / stride + 1, Wo = (W + 2 * pad - S) / stride + 1;
  LO_CHECK_ARG(Ho > 0 && Wo > 0, "empty output");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t work = (int64_t)N * H * W * (C / 8);
  LO_DISPATCH_DT(dt, T, (col2im_kernel<T><<<grid_for(work, 256), 256, 0, st>>>((const T*)dcol, (const T*)mask, (T*)dx, N, H, W, C, R, S,
                                                                                  stride, pad, Ho, Wo)));
  LO_LAUNCH_OK();
  return LO_OK;
}
int lo_transpose(const void* in, int64_t ld_in, void* out, int64_t ld_out, int dt, int K, int N, void* stream) {
  LO_CHECK_ARG(in && out && K > 0 && N > 0 && ld_in >= N && ld_out >= K, "null pointer / shape");
  cudaStream_t st = (cudaStream_t)stream;
  LO_DISPATCH_DT(dt, T, (transpose2d_kernel<T><<<dim3(cdiv(N, 32), cdiv(K, 32)), dim3(32, 8), 0, st>>>((const T*)in, ld_in, (T*)out, ld_out,
                                                                                                          K, N)));
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_conv3x3(const void* x, const void* w, const float* bias, const void* mask, void* y, int dt, int N, int H, int W,
               int Cin, int Cout, int pad, int relu, int impl, void* stream) {
  LO_CHECK_ARG(x && w && y, "null pointer");
  LO_CHECK_ARG(pad >= 0 && pad <= 2 && Cin % 16 == 0 && Cout % 8 == 0, "pad in 0..2, Cin%16==0, Cout%8==0");
  LO_CHECK_ARG(H + 2 * pad - 2 > 0 && W + 2 * pad - 2 > 0, "output would be empty");
  cudaStream_t st = (cudaStream_t)stream;
  if (impl == LO_IMPL_TC) {
    LO_CHECK_ARG(dt == LO_BF16, "wgmma path needs bf16 storage");
    if (!tc_available()) return fail(LO_ENOTSUP, "%s: wgmma path requires an sm_90 device", __func__);
    return tc_conv3x3((const bf16*)x, (const bf16*)w, bias, (const bf16*)mask, (bf16*)y, N, H, W, Cin, Cout, pad, relu, st);
  }
  const int Ho = H + 2 * pad - 2, Wo = W + 2 * pad - 2;
  const int64_t mtiles = ((int64_t)N * Ho * Wo + 63) / 64;
  LO_CHECK_ARG(mtiles <= INT32_MAX && Cout <= 64 * 65535, "shape (too many output positions or channels for the grid)");
  dim3 grid((unsigned)mtiles, cdiv(Cout, 64));
  LO_DISPATCH_DT(dt, T, (conv3x3_igemm_kernel<T><<<grid, 256, 0, st>>>((const T*)x, (const T*)w, bias, (const T*)mask, (T*)y,
                                                                       N, H, W, Cin, Cout, pad, relu)));
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_conv3x3_wgrad(const void* x, const void* dy, float* dw, float* db, int dt, int N, int H, int W, int Cin, int Cout,
                     int pad, int impl, void* stream) {
  LO_CHECK_ARG(x && dy && dw, "null pointer");
  LO_CHECK_ARG(pad >= 0 && pad <= 2 && Cin % 8 == 0 && Cout % 8 == 0, "shape");
  cudaStream_t st = (cudaStream_t)stream;
  const int Ho = H + 2 * pad - 2, Wo = W + 2 * pad - 2;
  const int64_t P = (int64_t)N * Ho * Wo;
  LO_CUDA(cudaMemsetAsync(dw, 0, (size_t)Cout * 9 * Cin * sizeof(float), st));
  if (impl == LO_IMPL_TC && dt == LO_BF16 && Cin % 64 == 0 && Cout % 128 == 0 && tc_available()) {
    LO_TRY(tc_conv3x3_wgrad((const bf16*)x, (const bf16*)dy, dw, N, H, W, Cin, Cout, pad, st));
    if (db) LO_TRY(colsum(dy, dt, db, (int)P, Cout, Cout, 0, st));
    return LO_OK;
  }
  // the splits add onto the zeroed dw with fp32 atomics.  Option "deterministic": at most two splits — two addends onto 0 sum
  // the same in either order (the rule of lo_gemm's split-K)
  const int tiles = 9 * cdiv(Cin, 64) * cdiv(Cout, 64);
  int splits = cdiv(LO_NUM_SMS * 4, tiles);
  const int maxs = (int)((P + 511) / 512);
  if (splits > maxs) splits = maxs;
  if (g_opt_det && splits > 2) splits = 2;
  if (splits < 1) splits = 1;
  dim3 grid(cdiv(Cin, 64), cdiv(Cout, 64), 9 * splits);
  LO_DISPATCH_DT(dt, T, (conv3x3_wgrad_kernel<T><<<grid, 256, 0, st>>>((const T*)x, (const T*)dy, dw, N, H, W, Cin, Cout, pad, splits)));
  LO_LAUNCH_OK();
  if (db) LO_TRY(colsum(dy, dt, db, (int)P, Cout, Cout, 0, st));
  return LO_OK;
}

int lo_conv_weight_flip(const void* w, void* wt, int dt, int Cin, int Cout, void* stream) {
  LO_CHECK_ARG(w && wt, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t total = (int64_t)Cin * 9 * Cout;
  LO_DISPATCH_DT(dt, T, (weight_flip_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)w, (T*)wt, Cin, Cout)));
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_maxpool_forward(const void* x, void* y, int dt, int N, int H, int W, int C, int kh, int kw, void* stream) {
  LO_CHECK_ARG(x && y && C % 8 == 0 && kh >= 1 && kw >= 1 && H >= kh && W >= kw, "shape");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t total = (int64_t)N * (H / kh) * (W / kw) * (C / 8);
  LO_DISPATCH_DT(dt, T, (maxpool_fwd_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)x, (T*)y, N, H, W, C, kh, kw)));
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_maxpool_backward(const void* x, const void* y, const void* dy, void* dx, int dt, int N, int H, int W, int C, int kh,
                        int kw, void* stream) {
  LO_CHECK_ARG(x && dy && dx && C % 8 == 0 && kh >= 1 && kw >= 1, "shape");
  (void)y;
  cudaStream_t st = (cudaStream_t)stream;
  if (H % kh || W % kw) LO_CUDA(cudaMemsetAsync(dx, 0, (size_t)N * H * W * C * (dt == LO_F32 ? 4 : 2), st));
  const int64_t total = (int64_t)N * (H / kh) * (W / kw) * (C / 8);
  LO_DISPATCH_DT(dt, T, (maxpool_bwd_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)x, (const T*)dy, (T*)dx, N, H, W, C, kh, kw)));
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_add_table(const void* y, const float* table, void* out, int dt, int N, int64_t HWC, void* stream) {
  LO_CHECK_ARG(y && table && out && HWC % 8 == 0, "shape");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t total8 = (int64_t)N * HWC / 8;
  LO_DISPATCH_DT(dt, T, (add_table_kernel<T><<<grid_for(total8, 256), 256, 0, st>>>((const T*)y, table, (T*)out, total8, HWC / 8)));
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_relu_mask_cast(const float* g, const void* y, void* out, int dt, int64_t n, void* stream) {
  LO_CHECK_ARG(g && y && out && n % 8 == 0, "shape");
  cudaStream_t st = (cudaStream_t)stream;
  LO_DISPATCH_DT(dt, T, (relu_mask_cast_kernel<T><<<grid_for(n / 8, 256), 256, 0, st>>>(g, (const T*)y, (T*)out, n / 8)));
  LO_LAUNCH_OK();
  return LO_OK;
}

}  // extern "C"
