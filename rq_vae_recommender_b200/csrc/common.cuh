// Shared device/host helpers for librqb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>

#define RQB_MAX_LEVELS 8

// ---- status codes of the C ABI (include/rqb200.h) ----
#define RQB_OK 0
#define RQB_ERR_INVALID 1      // bad argument (shape, alignment, null pointer)
#define RQB_ERR_CUDA 2         // a CUDA runtime call / launch failed
#define RQB_ERR_UNSUPPORTED 3  // shape outside what the kernels were built for
#define RQB_ERR_WORKSPACE 4    // workspace too small

void rqb_set_error(const char* fmt, ...);

#define RQB_CHECK_ARG(cond, ...)                  \
  do {                                            \
    if (!(cond)) {                                \
      rqb_set_error(__VA_ARGS__);                 \
      return RQB_ERR_INVALID;                     \
    }                                             \
  } while (0)

#define RQB_CUDA(call)                                                                     \
  do {                                                                                     \
    cudaError_t e__ = (call);                                                              \
    if (e__ != cudaSuccess) {                                                              \
      rqb_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      return RQB_ERR_CUDA;                                                                 \
    }                                                                                      \
  } while (0)

#define RQB_LAUNCH_CHECK() RQB_CUDA(cudaGetLastError())

static inline int64_t rqb_round_up(int64_t a, int64_t b) { return (a + b - 1) / b * b; }

#ifdef __CUDACC__
// ---------------------------------------------------------------- warp helpers
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// lexicographic (value, index) minimum: first index wins ties, like torch.min(dim).indices on CPU
__device__ __forceinline__ void warp_argmin(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, v, o);
    int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
}

// ---------------------------------------------------------------- mbarrier + bulk-copy (TMA) PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// same, but a wait longer than ~2 s (a protocol bug, never legitimate) traps instead of hanging the GPU.
// No printf here: it would force a stack frame and spills into the single-thread MMA / producer loops.
__device__ __forceinline__ void mbar_wait_guarded(uint64_t* bar, uint32_t parity, int /*tag*/) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
// ---- cluster variants
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// shared::cluster address of the same shared-memory offset in CTA `rank` of this cluster
__device__ __forceinline__ uint32_t cluster_map(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {   // every thread of every CTA of the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// distributed shared memory: loads, stores and atomics at a shared::cluster address (cluster_map)
__device__ __forceinline__ int ld_shared_cluster_s32(uint32_t cluster_addr) {
  int v;
  asm volatile("ld.shared::cluster.s32 %0, [%1];" : "=r"(v) : "r"(cluster_addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_cluster_u64(uint32_t cluster_addr, unsigned long long v) {
  asm volatile("st.shared::cluster.u64 [%0], %1;" ::"r"(cluster_addr), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t atom_add_shared_cluster_u32(uint32_t cluster_addr, uint32_t v) {
  uint32_t old;
  asm volatile("atom.shared::cluster.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(cluster_addr), "r"(v) : "memory");
  return old;
}
// arrive on an mbarrier anywhere in the cluster (own CTA included), release at cluster scope
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait_cluster(uint64_t* bar, uint32_t parity) {   // acquire at cluster scope
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_guarded_cluster(uint64_t* bar, uint32_t parity, int /*tag*/) {
  if (mbar_try_wait_cluster(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait_cluster(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}

// 1-D bulk async copy global -> shared (TMA engine, no tensor map): SASS UBLKCP
// fire-and-forget L2 prefetch of `bytes` (multiple of 16) from a 16-byte aligned global address
__device__ __forceinline__ void bulk_prefetch_l2(const void* gmem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// tiled tensor copy global -> shared of the box at (c0, c1) of a 2-D tensor map (a __grid_constant__ kernel parameter);
// 128-byte aligned destination.  SASS UTMALDG
__device__ __forceinline__ void tensor_g2s_2d(void* smem_dst, const void* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
#endif  // __CUDACC__
