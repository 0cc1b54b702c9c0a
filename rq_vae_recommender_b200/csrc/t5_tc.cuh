// TF32 wgmma helpers shared by the tensor-core attentions (csrc/t5enc_tc.cu, csrc/t5rank.cu): the K-major shared-memory tile
// layout without swizzle, its descriptors, the m64n64k8 TF32 MMAs and the staging copies (plain and transposing, the latter
// with each group of 8 keys in the order 0,2,4,6,1,3,5,7 so that an accumulator is the A fragment of the next product).
#pragma once
#include "common.cuh"

#define TC_T 64                  // rows per tile: queries or keys
#define TC_TILE (TC_T * 64)      // floats per staged 64 x 64 tile
#define TC_THREADS 128           // one warpgroup

// ------------------------------------------------------------------------------------------------ wgmma TF32 wrappers
// element (row r, k) of a 64 x 64 K-major tile without swizzle, in floats
__device__ __forceinline__ int tc_off(int r, int k) { return (r >> 3) * 512 + (k >> 2) * 32 + (r & 7) * 4 + (k & 3); }

// no-swizzle K-major descriptor of the tile at its K offset k0 (a multiple of 8): LBO 128 B, SBO 2048 B, layout 0
__device__ __forceinline__ uint64_t tc_desc(const float* tile, int k0) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(tile)) + k0 * 32;
  return (uint64_t)((a >> 4) & 0x3FFF) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(2048 >> 4) << 32);
}

__device__ __forceinline__ uint32_t tf32_bits(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float tf32(float x) { return __uint_as_float(tf32_bits(x)); }

__device__ __forceinline__ void tc_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tc_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tc_wait() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void tc_proxy_fence() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
template <typename T> __device__ __forceinline__ void tc_pin(T (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+r"(reinterpret_cast<uint32_t&>(d[i]))::"memory");
}

#define TC_D32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
               "%24, %25, %26, %27, %28, %29, %30, %31}"
#define TC_D32_OUT(d)                                                                                                            \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),        \
      "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),       \
      "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),       \
      "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// D[64 x 64] (+)= A[64 x 8] B[64 x 8]^T, both from shared memory; scale_d = 0 overwrites D
__device__ __forceinline__ void tc_mma_ss(float (&d)[32], uint64_t a, uint64_t b, int scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " TC_D32 ", %32, %33, p, 1, 1;\n\t}"
               : TC_D32_OUT(d)
               : "l"(a), "l"(b), "r"(scale_d));
}
// D += A B^T with A from registers: the TF32 fragment (row g, k t), (g + 8, t), (g, t + 4), (g + 8, t + 4)
__device__ __forceinline__ void tc_mma_rs(float (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t b) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " TC_D32 ", {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
               : TC_D32_OUT(d)
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b));
}

// D = A[64 x 64] B[64 x 64]^T over the tiles' whole K (eight k8 steps)
__device__ __forceinline__ void tc_gemm_ss(float (&d)[32], const float* a, const float* b) {
#pragma unroll
  for (int k = 0; k < 8; ++k) tc_mma_ss(d, tc_desc(a, 8 * k), tc_desc(b, 8 * k), k > 0);
}
// D += A B^T, A in the accumulator layout as TF32 bits (so the B tile's K runs in the permuted order)
__device__ __forceinline__ void tc_gemm_rs(float (&d)[32], const uint32_t (&a)[32], const float* b) {
#pragma unroll
  for (int k = 0; k < 8; ++k) tc_mma_rs(d, a[4 * k], a[4 * k + 2], a[4 * k + 1], a[4 * k + 3], tc_desc(b, 8 * k));
}

// ------------------------------------------------------------------------------------------------ staging copies
// rows 0 .. 63 of a row-major matrix (64 floats from `base`, row stride ld) as a K-major tile (row r, k = column), TF32-rounded;
// rows at or past nrows are zero and never read.  Thread i writes row group p, row i % 8, columns 4 ((i / 8) % 16) ..: a quarter
// warp writes one 128-byte core matrix.
__device__ __forceinline__ void tc_stage(float* tile, const float* base, int64_t ld, int nrows) {
  const int r0 = threadIdx.x & 7, c = (threadIdx.x >> 3) & 15;
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int r = p * 8 + r0;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < nrows) v = __ldg(reinterpret_cast<const float4*>(base + r * ld) + c);
    *reinterpret_cast<float4*>(tile + tc_off(r, 4 * c)) = make_float4(tf32(v.x), tf32(v.y), tf32(v.z), tf32(v.w));
  }
}

// position in the K order of a transposed tile -> the row it holds: 0,2,4,6,1,3,5,7 in each group of 8
__device__ __forceinline__ int tc_perm_row(int k) { return (k & ~7) | ((k & 4) ? 2 * (k & 3) + 1 : 2 * (k & 3)); }

// the transpose: tile row d (a column of the matrix), K position k holds matrix row tc_perm_row(k).  Lane l of a warp writes
// column 8 dhi + l % 8 at K position 4 kg + l / 8: the 32 lanes fill one 128-byte core-matrix row block without conflicts.
__device__ __forceinline__ void tc_stage_t(float* tile, const float* base, int64_t ld, int nrows) {
  const int dlo = threadIdx.x & 7, kq = (threadIdx.x >> 3) & 3, w = threadIdx.x >> 5;
#pragma unroll 8
  for (int p = 0; p < 32; ++p) {
    const int combo = p * 4 + w, dhi = combo & 7, kg = combo >> 3;
    const int j = tc_perm_row(kg * 4 + kq);
    const float v = j < nrows ? __ldg(base + j * ld + dhi * 8 + dlo) : 0.f;
    tile[dhi * 512 + kg * 32 + dlo * 4 + kq] = tf32(v);
  }
}
