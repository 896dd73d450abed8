// Fused Adam over one flat parameter buffer (torch.optim.Adam defaults, img2seq_torch.py:86-87,168-170)
// + dtype casts.  The step counter lives on the device so the call can be replayed inside a CUDA graph.
#include "lo_common.cuh"

namespace lo {

__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            bf16* __restrict__ shadow, int64_t n, const float* __restrict__ state, float b1, float b2, float eps,
                            float gscale) {
  const float step = state[0] + 1.0f;      // state[0] is bumped by adam_bump_kernel after this kernel
  const float lr = state[1];
  const float bc1 = 1.0f - powf(b1, step);
  const float bc2 = 1.0f - powf(b2, step);
  const float step_size = lr / bc1;
  const float inv_sqrt_bc2 = rsqrtf(bc2);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gi = g[i] * gscale;
    const float mi = b1 * m[i] + (1.0f - b1) * gi;
    const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) * inv_sqrt_bc2 + eps;
    const float pi = p[i] - step_size * (mi / denom);
    p[i] = pi;
    if (shadow) shadow[i] = __float2bfloat16_rn(pi);
  }
}
__global__ void adam_bump_kernel(float* state) { state[0] += 1.0f; }

// The optimisers the TF trainer offers (model/img2seq.py:98-111), TensorFlow 1.12 update rules and slot initial values:
//   kind 1  tf.train.AdamOptimizer            lr_t = lr sqrt(1-b2^t)/(1-b1^t) ; p -= lr_t m / (sqrt(v) + eps)   (eps OUTSIDE the bias correction)
//   kind 2  tf.train.GradientDescentOptimizer  p -= lr g
//   kind 3  tf.train.AdagradOptimizer          acc += g^2 (slot starts at 0.1) ; p -= lr g / sqrt(acc)
//   kind 4  tf.train.RMSPropOptimizer          ms = 0.9 ms + 0.1 g^2 (slot starts at 1) ; p -= lr g / sqrt(ms + 1e-10)   (momentum 0)
// s1 / s2 are the slot buffers (m, v | - | acc | ms); the host initialises them (FlatStore.ensure_optimizer).
__global__ void tf_optim_kernel(int kind, float* __restrict__ p, const float* __restrict__ g, float* __restrict__ s1, float* __restrict__ s2,
                                bf16* __restrict__ shadow, int64_t n, const float* __restrict__ state, float b1, float b2, float eps,
                                float gscale) {
  const float step = state[0] + 1.0f;
  const float lr = state[1];
  float lr_t = lr;
  if (kind == 1) lr_t = lr * sqrtf(1.0f - powf(b2, step)) / (1.0f - powf(b1, step));
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gi = g[i] * gscale;
    float pi = p[i];
    if (kind == 1) {
      const float mi = b1 * s1[i] + (1.0f - b1) * gi;
      const float vi = b2 * s2[i] + (1.0f - b2) * gi * gi;
      s1[i] = mi;
      s2[i] = vi;
      pi -= lr_t * mi / (sqrtf(vi) + eps);
    } else if (kind == 2) {
      pi -= lr * gi;
    } else if (kind == 3) {
      const float a = s1[i] + gi * gi;
      s1[i] = a;
      pi -= lr * gi * rsqrtf(a);
    } else {
      const float ms = b2 * s1[i] + (1.0f - b2) * gi * gi;      // b2 carries the decay (0.9)
      s1[i] = ms;
      pi -= lr * gi * rsqrtf(ms + eps);
    }
    p[i] = pi;
    if (shadow) shadow[i] = __float2bfloat16_rn(pi);
  }
}

template <typename TS, typename TD>
__global__ void cast_kernel(const TS* __restrict__ s, TD* __restrict__ d, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) stf(d + i, ldf(s + i));
}

}  // namespace lo

using namespace lo;

extern "C" {

int lo_adam_step(float* p, const float* g, float* m, float* v, void* shadow_bf16, int64_t n, float* state_dev, float beta1,
                 float beta2, float eps, float grad_scale, void* stream) {
  LO_CHECK_ARG(p && g && m && v && state_dev && n > 0, "null pointer / n");
  cudaStream_t st = (cudaStream_t)stream;
  int grid = (int)((n + 1023) / 1024);
  if (grid > LO_NUM_SMS * 8) grid = LO_NUM_SMS * 8;
  adam_kernel<<<grid, 256, 0, st>>>(p, g, m, v, (bf16*)shadow_bf16, n, state_dev, beta1, beta2, eps, grad_scale);
  LO_LAUNCH_OK();
  adam_bump_kernel<<<1, 1, 0, st>>>(state_dev);
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_adam_step_ranges(float* p, const float* g, float* m, float* v, void* shadow_bf16, const int64_t* ranges, int n_ranges,
                        float* state_dev, float beta1, float beta2, float eps, float grad_scale, void* stream) {
  LO_CHECK_ARG(p && g && m && v && state_dev && ranges && n_ranges >= 0, "null pointer / n_ranges");
  cudaStream_t st = (cudaStream_t)stream;
  for (int r = 0; r < n_ranges; r++) {
    const int64_t off = ranges[2 * r], n = ranges[2 * r + 1];
    LO_CHECK_ARG(off >= 0 && n > 0, "range");
    int grid = (int)((n + 1023) / 1024);
    if (grid > LO_NUM_SMS * 8) grid = LO_NUM_SMS * 8;
    adam_kernel<<<grid, 256, 0, st>>>(p + off, g + off, m + off, v + off, shadow_bf16 ? (bf16*)shadow_bf16 + off : nullptr, n, state_dev, beta1,
                                      beta2, eps, grad_scale);
    LO_LAUNCH_OK();
  }
  adam_bump_kernel<<<1, 1, 0, st>>>(state_dev);
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_tf_optim_step(int kind, float* p, const float* g, float* s1, float* s2, void* shadow_bf16, int64_t n, float* state_dev, float beta1,
                     float beta2, float eps, float grad_scale, void* stream) {
  LO_CHECK_ARG(p && g && state_dev && n > 0, "null pointer / n");
  LO_CHECK_ARG(kind >= 1 && kind <= 4, "kind: 1 Adam (TF epsilon), 2 SGD, 3 Adagrad, 4 RMSProp");
  LO_CHECK_ARG((kind != 1 || (s1 && s2)) && (kind < 3 || s1), "slot buffers");
  cudaStream_t st = (cudaStream_t)stream;
  int grid = (int)((n + 1023) / 1024);
  if (grid > LO_NUM_SMS * 8) grid = LO_NUM_SMS * 8;
  tf_optim_kernel<<<grid, 256, 0, st>>>(kind, p, g, s1, s2, (bf16*)shadow_bf16, n, state_dev, beta1, beta2, eps, grad_scale);
  LO_LAUNCH_OK();
  adam_bump_kernel<<<1, 1, 0, st>>>(state_dev);
  LO_LAUNCH_OK();
  return LO_OK;
}

int lo_cast(const void* src, int dt_src, void* dst, int dt_dst, int64_t n, void* stream) {
  LO_CHECK_ARG(src && dst && n > 0, "null pointer / n");
  cudaStream_t st = (cudaStream_t)stream;
  int grid = (int)((n + 1023) / 1024);
  if (grid > LO_NUM_SMS * 8) grid = LO_NUM_SMS * 8;
  if (dt_src == LO_F32 && dt_dst == LO_BF16) cast_kernel<float, bf16><<<grid, 256, 0, st>>>((const float*)src, (bf16*)dst, n);
  else if (dt_src == LO_BF16 && dt_dst == LO_F32) cast_kernel<bf16, float><<<grid, 256, 0, st>>>((const bf16*)src, (float*)dst, n);
  else if (dt_src == LO_F32 && dt_dst == LO_F32) cast_kernel<float, float><<<grid, 256, 0, st>>>((const float*)src, (float*)dst, n);
  else if (dt_src == LO_BF16 && dt_dst == LO_BF16) cast_kernel<bf16, bf16><<<grid, 256, 0, st>>>((const bf16*)src, (bf16*)dst, n);
  else return fail(LO_EINVAL, "%s: bad dtype", __func__);
  LO_LAUNCH_OK();
  return LO_OK;
}

}  // extern "C"
