// Inline-PTX wrappers shared by the TMA/mbarrier kernels (strings follow cute/arch/copy_sm90_tma.hpp, cutlass/arch/barrier.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lo {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}\n"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  // fast path: no clock reads.  try_wait suspends for a bounded time per call; a wait that never completes traps
  // (after ~2 s) instead of hanging the GPU — a protocol bug must fail loudly.
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// 1-D bulk copy global -> shared (TMA engine, no tensor map), completion on an mbarrier, with an L2 cache policy
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_normal() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// Programmatic dependent launch: a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may become
// resident while its predecessor is still running.  pdl_wait() returns once every prerequisite grid has completed and
// its writes are visible — it must precede ANY global-memory access; pdl_trigger() lets the successor start launching.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Deterministic cross-CTA sums: the CTAs that contribute to the same outputs form one thread-block cluster, each stages its
// partial sums at the same shared-memory offset, and rank 0 adds them in rank order (distributed shared memory) before the
// single write to global memory — no fp32 atomics whose order, and so whose rounding, changes from run to run.
// Every thread of every CTA of the cluster must call cl_sync() (no early exit before the last one).
__device__ __forceinline__ uint32_t cl_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cl_size() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cl_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the two halves of cl_sync(), for work in between that touches no peer's shared memory
__device__ __forceinline__ void cl_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cl_wait_acquire() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
// the float at the same shared-memory offset as `p` in CTA `rank` of the cluster
__device__ __forceinline__ float cl_ld(const float* p, uint32_t rank) {
  uint32_t a;
  float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(smem_u32(p)), "r"(rank));
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
  return v;
}
// sum over the cluster's CTAs (<= 16), in rank order, of the float at `p`; all loads are issued before the first add
__device__ __forceinline__ float cl_sum(const float* p) {
  const uint32_t n = cl_size();
  float v[16];
#pragma unroll
  for (uint32_t r = 0; r < 16; r++) v[r] = r < n ? cl_ld(p, r) : 0.f;
  float s = v[0];
#pragma unroll
  for (uint32_t r = 1; r < 16; r++)
    if (r < n) s += v[r];
  return s;
}
// out[i] = the same sum for the K floats at p + i * stride; the K loads of one rank are in flight together
template <int K>
__device__ __forceinline__ void cl_sum_n(const float* p, int stride, float* out) {
  const uint32_t n = cl_size();
#pragma unroll
  for (int i = 0; i < K; i++) out[i] = cl_ld(p + i * stride, 0);
  for (uint32_t r = 1; r < n; r++) {
    float v[K];
#pragma unroll
    for (int i = 0; i < K; i++) v[i] = cl_ld(p + i * stride, r);
#pragma unroll
    for (int i = 0; i < K; i++) out[i] += v[i];
  }
}

}  // namespace lo
