// bf16 wgmma GEMM with fused ReLU for the encoder / decoder MLPs (modules/encoder.py:23-38), sm_90a.
//
//   Y[M,N] = act( X[M,K] . W[N,K]^T ),   bf16 operands, fp32 accumulation in registers, act = ReLU or identity.
//
// This is the reduced-precision (AMP-like) path: the reference runs these Linears in bf16 when
// `train_rqvae.py:36,69` enables mixed precision.  The exact fp32 path (csrc/dense.cu sgemm) stays the default because
// index parity at 1e-5 needs it; this kernel is opt-in and forward-only (tokenisation).
//
// Data layout ("image"): every operand is stored in HBM as the exact shared-memory image the tensor core reads --
// [row-tile of 128][k-chunk of 64][128 rows x 128 B], K-major, 16-byte chunks XOR-swizzled with (row & 7) (wgmma
// SWIZZLE_128B).  A stage is then ONE contiguous 16 KB bulk copy, no tensor maps, and the epilogue of layer i
// writes layer i+1's A operand directly in that layout, so activations never exist in row-major form.
//
// Kernel: persistent, one CTA per SM.  warps 0-7 = two consumer warpgroups (rows [0,64) and [64,128) of the tile, wgmma
// m64n128k16 per 128-column W block, accumulators in registers), warp 8 = bulk-copy producer (A + up to 2 W blocks per stage,
// 4-stage ring).  The epilogue (ReLU -> bf16 image or fp32 rows) runs from the accumulator registers.
#include "common.cuh"
#include "wgmma.cuh"
#include <cuda_bf16.h>

#define GT_KC 64
#define GT_BLK_BYTES (128 * GT_KC * 2)   // 16 KB: 128 rows x 64 bf16
#define GT_STAGES 4
#define GT_THREADS 288                   // warps 0-7: two consumer warpgroups | warp 8: producer

// ------------------------------------------------------------------------------------------------ image builders
extern "C" size_t rqb200_bf16_image_bytes(int rows, int K) {
  if (rows < 0 || K <= 0 || K % GT_KC) return 0;
  return (size_t)((rows + 127) / 128) * (K / GT_KC) * GT_BLK_BYTES;
}

// fp32 row-major [rows, K] -> bf16 image; rows beyond `rows` in the last tile are zero.  One CTA per (row tile, k chunk).
__global__ void gt_f32_to_image_kernel(const float* __restrict__ x, int64_t ldx, int rows, int K, __nv_bfloat16* img) {
  const int nkc = K / GT_KC;
  const int mt = blockIdx.x / nkc, kc = blockIdx.x % nkc;
  unsigned char* out = reinterpret_cast<unsigned char*>(img) + (size_t)blockIdx.x * GT_BLK_BYTES;
  for (int i = threadIdx.x; i < 128 * 8; i += blockDim.x) {
    const int r = i >> 3, c = i & 7;              // row in tile, 16-byte chunk (8 elements)
    const int row = mt * 128 + r;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
    if (row < rows) {
      const float* src = x + (int64_t)row * ldx + kc * GT_KC + c * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = __ldg(src + e);
    }
    __nv_bfloat162 p0 = __floats2bfloat162_rn(v[0], v[1]), p1 = __floats2bfloat162_rn(v[2], v[3]);
    __nv_bfloat162 p2 = __floats2bfloat162_rn(v[4], v[5]), p3 = __floats2bfloat162_rn(v[6], v[7]);
    uint4 w;
    w.x = *reinterpret_cast<uint32_t*>(&p0); w.y = *reinterpret_cast<uint32_t*>(&p1);
    w.z = *reinterpret_cast<uint32_t*>(&p2); w.w = *reinterpret_cast<uint32_t*>(&p3);
    *reinterpret_cast<uint4*>(out + r * 128 + ((c ^ (r & 7)) << 4)) = w;
  }
}

extern "C" int rqb200_f32_to_bf16_image(const float* x, int64_t ldx, int rows, int K, void* image, void* stream) {
  RQB_CHECK_ARG(K > 0 && K % GT_KC == 0 && rows >= 0 && ldx >= K, "f32_to_bf16_image: need K %% 64 == 0 (K=%d)", K);
  if (rows == 0) return RQB_OK;
  RQB_CHECK_ARG(x && image, "f32_to_bf16_image: null pointer");
  const int blocks = ((rows + 127) / 128) * (K / GT_KC);
  gt_f32_to_image_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, ldx, rows, K, reinterpret_cast<__nv_bfloat16*>(image));
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ------------------------------------------------------------------------------------------------ GEMM
struct GtParams {
  const unsigned char* a_img;   // [mtiles][nkc][16 KB]
  const unsigned char* w_img;   // [nblocks][nkc][16 KB]   (rows of W padded with zeros to a multiple of 128)
  int M, N, K, nkc, mtiles, nblocks, ngroups, nitems;
  int relu;
  unsigned char* out_img;       // next layer's A image [mtiles][N/64][16 KB] (N % 64 == 0), or null
  float* out_f32;               // row-major [M, N] (ld = ldo), or null
  int64_t ldo;
};

struct GtSmemMisc {
  uint64_t full[GT_STAGES], empty[GT_STAGES];
};

// one 128-column block of the epilogue: columns col0 + 8 jb + 2 (lane % 4) + {0, 1} of rows ra and ra + 8 (acc[4 jb + 0..3])
__device__ __forceinline__ void gt_store_block(const GtParams& p, const float (&acc)[64], int mt, int ra, int col0, int lane) {
  const int q4 = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = ra + 8 * h, row = mt * 128 + r;
#pragma unroll
    for (int jb = 0; jb < 16; ++jb) {
      const int col = col0 + 8 * jb + 2 * q4;
      if (col >= p.N) continue;
      float v0 = acc[4 * jb + 2 * h], v1 = acc[4 * jb + 2 * h + 1];
      if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      if (p.out_img) {
        // next layer's A image (N % 64 == 0, so col + 1 < N): rows >= M hold act(0) = 0, harmless padding
        unsigned char* dst = p.out_img + ((size_t)mt * (p.N / GT_KC) + (col >> 6)) * GT_BLK_BYTES + r * 128 +
                             ((((col & 63) >> 3) ^ (r & 7)) << 4) + (col & 7) * 2;
        *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v0, v1);
      }
      if (p.out_f32 && row < p.M) {
        float* o = p.out_f32 + (int64_t)row * p.ldo + col;
        o[0] = v0;
        if (col + 1 < p.N) o[1] = v1;
      }
    }
  }
}

__global__ void __launch_bounds__(GT_THREADS, 1) gt_gemm_kernel(GtParams p) {
  extern __shared__ __align__(1024) unsigned char gsm[];
  // stage s: [A 16 KB][W block 0 16 KB][W block 1 16 KB]
  GtSmemMisc* ms = reinterpret_cast<GtSmemMisc*>(gsm + GT_STAGES * 3 * GT_BLK_BYTES);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    if ((smem_u32(gsm) & 1023u) != 0) __trap();
    for (int i = 0; i < GT_STAGES; ++i) { mbar_init(&ms->full[i], 1); mbar_init(&ms->empty[i], 8); }
    fence_mbar_init();
  }
  __syncthreads();

  // work item = (row tile mt, group of up to two 128-column W blocks)
  if (warp == 8) {
    // ============================================================== bulk-copy producer
    if (lane == 0) {
      uint32_t s = 0;
      for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
        const int mt = item / p.ngroups, g = item % p.ngroups;
        const int nb = min(2, p.nblocks - 2 * g);
        for (int kc = 0; kc < p.nkc; ++kc, ++s) {
          const uint32_t st = s % GT_STAGES, u = s / GT_STAGES;
          mbar_wait_guarded(&ms->empty[st], (u & 1) ^ 1, 1);
          unsigned char* dst = gsm + st * 3 * GT_BLK_BYTES;
          mbar_expect_tx(&ms->full[st], (1 + nb) * GT_BLK_BYTES);
          bulk_g2s(dst, p.a_img + ((size_t)mt * p.nkc + kc) * GT_BLK_BYTES, GT_BLK_BYTES, &ms->full[st]);
          for (int b = 0; b < nb; ++b)
            bulk_g2s(dst + (1 + b) * GT_BLK_BYTES, p.w_img + ((size_t)(2 * g + b) * p.nkc + kc) * GT_BLK_BYTES, GT_BLK_BYTES,
                     &ms->full[st]);
        }
      }
    }
    return;
  }
  // ============================================================== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64)
  const int wg = warp >> 2;
  const int ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const uint32_t base = smem_u32(gsm);
  uint32_t s = 0;
  for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
    const int mt = item / p.ngroups, g = item % p.ngroups;
    const int nb = min(2, p.nblocks - 2 * g);
    float acc0[64], acc1[64];
    uint32_t prev = 0;
    for (int kc = 0; kc < p.nkc; ++kc, ++s) {
      const uint32_t st = s % GT_STAGES;
      mbar_wait_guarded(&ms->full[st], (s / GT_STAGES) & 1, 3);
      const uint32_t sa = base + st * 3 * GT_BLK_BYTES;
      const uint64_t ad = wg_desc(sa + wg * (GT_BLK_BYTES / 2)), b0 = wg_desc(sa + GT_BLK_BYTES), b1 = wg_desc(sa + 2 * GT_BLK_BYTES);
      wg_fence_acc(acc0); wg_fence_acc(acc1);
      wg_fence();
#pragma unroll
      for (int j = 0; j < GT_KC / 16; ++j) {
        // the second block is multiplied even when the group has one (its stale slot is never stored): a wgmma under a
        // branch is serialised by the compiler
        wg_m64n128_bf16(acc0, ad + 2 * j, b0 + 2 * j, (kc | j) != 0);
        wg_m64n128_bf16(acc1, ad + 2 * j, b1 + 2 * j, (kc | j) != 0);
      }
      wg_commit();
      wg_fence_acc(acc0); wg_fence_acc(acc1);
      if (kc > 0) {
        wg_wait<1>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&ms->empty[prev]);
      }
      prev = st;
    }
    wg_wait<0>();
    wg_fence_acc(acc0); wg_fence_acc(acc1);
    __syncwarp();
    if (lane == 0) mbar_arrive(&ms->empty[prev]);
    gt_store_block(p, acc0, mt, ra, 2 * g * 128, lane);
    if (nb > 1) gt_store_block(p, acc1, mt, ra, (2 * g + 1) * 128, lane);
  }
}

extern "C" int rqb200_gemm_bf16(const void* a_image, const void* w_image, int M, int N, int K, int relu, void* out_image,
                                float* out_f32, int64_t ldo, void* stream) {
  RQB_CHECK_ARG(M >= 0 && N > 0 && K > 0 && K % GT_KC == 0, "gemm_bf16: need K %% 64 == 0 (M=%d N=%d K=%d)", M, N, K);
  RQB_CHECK_ARG(!out_image || N % GT_KC == 0, "gemm_bf16: an image output needs N %% 64 == 0 (N=%d)", N);
  RQB_CHECK_ARG(out_image || out_f32, "gemm_bf16: no output");
  RQB_CHECK_ARG(!out_f32 || ldo >= N, "gemm_bf16: ldo < N");
  if (M == 0) return RQB_OK;
  RQB_CHECK_ARG(a_image && w_image, "gemm_bf16: null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  GtParams p{};
  p.a_img = reinterpret_cast<const unsigned char*>(a_image);
  p.w_img = reinterpret_cast<const unsigned char*>(w_image);
  p.M = M; p.N = N; p.K = K; p.nkc = K / GT_KC;
  p.mtiles = (M + 127) / 128;
  p.nblocks = (N + 127) / 128;
  p.ngroups = (p.nblocks + 1) / 2;
  p.nitems = p.mtiles * p.ngroups;
  p.relu = relu;
  p.out_img = reinterpret_cast<unsigned char*>(out_image);
  p.out_f32 = out_f32; p.ldo = ldo;
  int dev = 0, sm_count = 0;                                 // per call: the current device may differ between calls
  RQB_CUDA(cudaGetDevice(&dev));
  RQB_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
  const size_t smem = (size_t)GT_STAGES * 3 * GT_BLK_BYTES + sizeof(GtSmemMisc);
  RQB_CUDA(cudaFuncSetAttribute(gt_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = p.nitems < sm_count ? p.nitems : sm_count;
  gt_gemm_kernel<<<grid, GT_THREADS, smem, st>>>(p);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// =====================================================================================================================
// Split-precision GEMM: fp32-accurate products on the fp16 tensor cores (the MLPs of modules/encoder.py:23-38 in their
// default, index-exact precision; the two GEMMs of a Gumbel-softmax level, modules/quantize.py:113-117,135).
//
//   C[M,N] = act( A[M,K] . B[N,K]^T ),  A, B, C fp32 in HBM.
//
// Every operand row is scaled by a power of two so that its largest element lies in [2^14, 2^15) and stored as TWO fp16 images
//   hi = fp16(v 2^e),  lo = fp16(v 2^e - hi)          (hi + lo carries 22 significant bits of v; lo may be subnormal: the error
//                                                      is then 2^-25 absolute = 2^-39 of the row maximum)
// and the product is three wgmma per k-step, hi.hi + lo.hi + hi.lo, each 64-wide k chunk promoted into an fp32 total (lo.lo is 2^-22
// relative and dropped).  The epilogue multiplies by 2^-(e_row + e_col), both exact.  Measured against float64 the result is
// as close as a plain fp32 FMA GEMM (tests/test_gpu_gemm_split.py states the bound that is asserted).  Below K = 64 a plain fp32
// GEMM is nearly exact and the format's worst case per product, 3 x 2^-22 of |a||b|, is the bound (tests/test_gpu_gemm_shapes.py).
//
// Image = the bf16 image's layout with fp16 elements: [row tile of 128][k chunk of 64][128 rows x 128 B swizzled]; one buffer
// holds [hi image][lo image][row scales: 128 floats per row tile, value 2^-e].  K is padded with zeros to a multiple of 64, rows
// to a multiple of 128.
//
// Kernel: persistent, one CTA per SM; work item = (row tile, 128-column block, k slice).  Stage = [A hi][A lo][B hi][B lo]
// = 64 KB, 3 stages.  warps 0-7 = two consumer warpgroups (64 rows each: an m64n128 register accumulator per k chunk, promoted
// into an fp32 total; the epilogue scales and activates), warp 8 = bulk-copy producer.
#include <cuda_fp16.h>

#define GS_STAGES 3
#define GS_MAX_CHUNKS 12                   // 16-byte chunks per lane of the row splitter: K <= 32 * 8 * 12 = 3072 (wider: two passes)
#define GS_STAGE_BYTES (4 * GT_BLK_BYTES)

extern "C" size_t rqb200_split_image_bytes(int rows, int K) {
  if (rows < 0 || K <= 0) return 0;
  const size_t mt = (size_t)(rows + 127) / 128, nkc = (size_t)(K + GT_KC - 1) / GT_KC;
  return 2 * mt * nkc * GT_BLK_BYTES + mt * 128 * sizeof(float);
}

__device__ __forceinline__ float gs_pow2_scale(float mx) {
  // 2^e with mx 2^e in [2^14, 2^15); zero / non-finite rows are not scaled
  if (!(mx > 0.f) || !(mx < INFINITY)) return 1.f;
  int ex;
  frexpf(mx, &ex);                        // mx = f 2^ex, f in [0.5, 1)
  return ldexpf(1.f, max(-120, min(120, 15 - ex)));      // (clamped: 2^e and 2^-e both stay normal)
}
__device__ __forceinline__ void gs_split8(const float (&v)[8], float s, uint4& hi, uint4& lo) {
  __half2 h[4], l[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float a = v[2 * e] * s, b = v[2 * e + 1] * s;
    h[e] = __floats2half2_rn(a, b);
    const float2 hf = __half22float2(h[e]);
    l[e] = __floats2half2_rn(a - hf.x, b - hf.y);
  }
  hi.x = *reinterpret_cast<uint32_t*>(&h[0]); hi.y = *reinterpret_cast<uint32_t*>(&h[1]);
  hi.z = *reinterpret_cast<uint32_t*>(&h[2]); hi.w = *reinterpret_cast<uint32_t*>(&h[3]);
  lo.x = *reinterpret_cast<uint32_t*>(&l[0]); lo.y = *reinterpret_cast<uint32_t*>(&l[1]);
  lo.z = *reinterpret_cast<uint32_t*>(&l[2]); lo.w = *reinterpret_cast<uint32_t*>(&l[3]);
}

// Row-major source [rows, K] (ld = ldx): W lanes per image row (32 / W rows per warp pass), NCH 16-byte chunks per lane; the row
// stays in registers between the maximum and the split.  grid = row tiles, block = 256.  Few registers on purpose: the kernel
// is a pure HBM stream (read 4 B, write 4 B per element) and needs many warps per SM in flight -- the first version (one
// generic 12-chunk instantiation, 133 registers, one CTA per SM) ran at 0.8-2 TB/s.
// LIVE (rqb200_f32_to_split_image_counted): the grid and image are sized for `rows` (the capacity) and the source rows are the
// first min(*live, rows): the CTAs of tiles past them exit, the rest write what a call with that row count writes.
template <int NCH, int W, bool LIVE>
__global__ void __launch_bounds__(256) gs_split_rows_kernel(const float* __restrict__ x, int64_t ldx, int rows, int K, unsigned char* img,
                                                            const int* __restrict__ live) {
  const int nkc = (K + GT_KC - 1) / GT_KC, mtiles = gridDim.x;
  const int mt = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (LIVE) {
    rows = min(rows, max(0, *live));
    if (mt * 128 >= rows) return;
  }
  unsigned char* hi_img = img;
  unsigned char* lo_img = img + (size_t)mtiles * nkc * GT_BLK_BYTES;
  float* scales = reinterpret_cast<float*>(img + 2 * (size_t)mtiles * nkc * GT_BLK_BYTES);
  const int nchunks = nkc * 8;                                    // 16-byte (8 element) chunks per image row
  const bool vec = (K % 8 == 0) && (ldx % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  constexpr int G = 32 / W;                                       // rows per warp pass
  const int sub = lane / W, sl = lane % W;
#pragma unroll 1
  for (int r = warp * G + sub; r < 128; r += 8 * G) {
    const int row = mt * 128 + r;
    float v[NCH][8];
    float mx = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = sl + W * i;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[i][e] = 0.f;
      if (c < nchunks && row < rows) {
        const float* src = x + (int64_t)row * ldx + c * 8;
        if (vec && c * 8 + 8 <= K) {
          const float4 a = __ldg(reinterpret_cast<const float4*>(src)), b = __ldg(reinterpret_cast<const float4*>(src) + 1);
          v[i][0] = a.x; v[i][1] = a.y; v[i][2] = a.z; v[i][3] = a.w; v[i][4] = b.x; v[i][5] = b.y; v[i][6] = b.z; v[i][7] = b.w;
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (c * 8 + e < K) v[i][e] = __ldg(src + e);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) mx = fmaxf(mx, fabsf(v[i][e]));
      }
    }
#pragma unroll
    for (int o = W / 2; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float s = gs_pow2_scale(mx);
    if (sl == 0) scales[mt * 128 + r] = 1.f / s;                   // exact: a power of two
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = sl + W * i;
      if (c < nchunks) {
        uint4 hi, lo;
        gs_split8(v[i], s, hi, lo);
        const size_t off = ((size_t)mt * nkc + (c >> 3)) * GT_BLK_BYTES + r * 128 + (((c & 7) ^ (r & 7)) << 4);
        *reinterpret_cast<uint4*>(hi_img + off) = hi;
        *reinterpret_cast<uint4*>(lo_img + off) = lo;
      }
    }
  }
}

// Rows wider than the register-resident splitter takes (K > 32 * 8 * GS_MAX_CHUNKS): one warp per image row, two passes over
// the row -- its maximum, then the split (the second read comes from L2: at most 8 rows of a CTA are in flight).  Same image
// and scale as gs_split_rows_kernel.  grid = 16 per row tile (8 rows each), block = 256.  LIVE as gs_split_rows_kernel.
template <bool LIVE>
__global__ void __launch_bounds__(256) gs_split_rows_wide_kernel(const float* __restrict__ x, int64_t ldx, int rows, int K,
                                                                 unsigned char* img, const int* __restrict__ live) {
  const int nkc = (K + GT_KC - 1) / GT_KC, mtiles = gridDim.x / 16;
  const int mt = blockIdx.x / 16, r = (blockIdx.x % 16) * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (LIVE) {
    rows = min(rows, max(0, *live));
    if (mt * 128 >= rows) return;
  }
  const int row = mt * 128 + r;
  unsigned char* hi_img = img;
  unsigned char* lo_img = img + (size_t)mtiles * nkc * GT_BLK_BYTES;
  float* scales = reinterpret_cast<float*>(img + 2 * (size_t)mtiles * nkc * GT_BLK_BYTES);
  const int nchunks = nkc * 8;
  const bool vec = (K % 8 == 0) && (ldx % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  // chunk c of the row (zeros past K and for rows >= rows): the splitters' 16-byte loads, or scalar loads off the vec layout
  auto load = [&](int c, float (&v)[8]) {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
    if (row >= rows) return;
    const float* src = x + (int64_t)row * ldx + c * 8;
    if (vec && c * 8 + 8 <= K) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(src)), b = __ldg(reinterpret_cast<const float4*>(src) + 1);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (c * 8 + e < K) v[e] = __ldg(src + e);
    }
  };
  float mx = 0.f;
  for (int c = lane; c < nchunks; c += 32) {
    float v[8];
    load(c, v);
#pragma unroll
    for (int e = 0; e < 8; ++e) mx = fmaxf(mx, fabsf(v[e]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  const float s = gs_pow2_scale(mx);
  if (lane == 0) scales[row] = 1.f / s;                          // exact: a power of two
  for (int c = lane; c < nchunks; c += 32) {
    float v[8];
    load(c, v);
    uint4 hi, lo;
    gs_split8(v, s, hi, lo);
    const size_t off = ((size_t)mt * nkc + (c >> 3)) * GT_BLK_BYTES + r * 128 + (((c & 7) ^ (r & 7)) << 4);
    *reinterpret_cast<uint4*>(hi_img + off) = hi;
    *reinterpret_cast<uint4*>(lo_img + off) = lo;
  }
}

// Transposed source: image row r = column r of x[K, rows] (ld = ldx) -- the operand of x^T without materialising the transpose
// (W^T for dgrad, C^T for W@C, g^T and h^T for the weight gradients whose contraction runs over the batch).  Three launches:
//   gs_colmax_kernel    |column| maxima by atomicMax on the float bits (non-negative floats order like unsigned ints) into scales[]
//   gs_colscale_kernel  scales[r] = 2^-e
//   gs_split_cols_kernel one CTA per (row tile, k chunk): 64 x 128 source floats through shared memory (coalesced reads, the
//                       transposed reads are conflict-free with a 129-float pitch), hi / lo blocks written as 16-byte chunks
__global__ void gs_colmax_kernel(const float* __restrict__ x, int64_t ldx, int rows, int K, unsigned int* colmax) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int k0 = blockIdx.y * 128;
  if (c >= rows) return;
  float mx = 0.f;
  const int k1 = min(K, k0 + 128);
  for (int k = k0; k < k1; ++k) mx = fmaxf(mx, fabsf(__ldg(x + (int64_t)k * ldx + c)));
  if (mx != mx) mx = INFINITY;                               // NaN: not scaled (gs_pow2_scale), like the row kernel
  atomicMax(colmax + c, __float_as_uint(mx));
}
__global__ void gs_colscale_kernel(float* scales, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) scales[i] = 1.f / gs_pow2_scale(scales[i]);
}
__global__ void __launch_bounds__(256) gs_split_cols_kernel(const float* __restrict__ x, int64_t ldx, int rows, int K, unsigned char* img) {
  __shared__ float tile[GT_KC][129];
  const int mtiles = gridDim.x, nkc = gridDim.y;
  const int mt = blockIdx.x, kc = blockIdx.y, t = threadIdx.x;
  unsigned char* hi_img = img;
  unsigned char* lo_img = img + (size_t)mtiles * nkc * GT_BLK_BYTES;
  const float* scales = reinterpret_cast<const float*>(img + 2 * (size_t)mtiles * nkc * GT_BLK_BYTES);
#pragma unroll 4
  for (int i = 0; i < (GT_KC * 128) / 256; ++i) {
    const int idx = t + 256 * i, kr = idx >> 7, c = idx & 127;
    const int k = kc * GT_KC + kr, row = mt * 128 + c;
    tile[kr][c] = (k < K && row < rows) ? __ldg(x + (int64_t)k * ldx + row) : 0.f;
  }
  __syncthreads();
  const int r = t & 127;
  const float s = 1.f / scales[mt * 128 + r];                 // exact: a power of two
#pragma unroll
  for (int cc = 0; cc < 4; ++cc) {
    const int c = (t >> 7) * 4 + cc;                          // 16-byte chunk of the 128-byte block row
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = tile[c * 8 + e][r];
    uint4 hi, lo;
    gs_split8(v, s, hi, lo);
    const size_t off = ((size_t)mt * nkc + kc) * GT_BLK_BYTES + r * 128 + ((c ^ (r & 7)) << 4);
    *reinterpret_cast<uint4*>(hi_img + off) = hi;
    *reinterpret_cast<uint4*>(lo_img + off) = lo;
  }
}

// the row-major splitter for K: the register-resident kernel whose lanes cover a row, or the two-pass one past 32 * 8 * GS_MAX_CHUNKS
template <bool LIVE>
static void gs_split_rows(const float* x, int64_t ldx, int rows, int K, unsigned char* im, const int* live, cudaStream_t st) {
  const int mtiles = (rows + 127) / 128, nchunks = ((K + GT_KC - 1) / GT_KC) * 8;
  if (nchunks <= 8) gs_split_rows_kernel<1, 8, LIVE><<<mtiles, 256, 0, st>>>(x, ldx, rows, K, im, live);
  else if (nchunks <= 16) gs_split_rows_kernel<1, 16, LIVE><<<mtiles, 256, 0, st>>>(x, ldx, rows, K, im, live);
  else if (nchunks <= 32) gs_split_rows_kernel<1, 32, LIVE><<<mtiles, 256, 0, st>>>(x, ldx, rows, K, im, live);
  else if (nchunks <= 64) gs_split_rows_kernel<2, 32, LIVE><<<mtiles, 256, 0, st>>>(x, ldx, rows, K, im, live);
  else if (nchunks <= 96) gs_split_rows_kernel<3, 32, LIVE><<<mtiles, 256, 0, st>>>(x, ldx, rows, K, im, live);
  else if (nchunks <= 128) gs_split_rows_kernel<4, 32, LIVE><<<mtiles, 256, 0, st>>>(x, ldx, rows, K, im, live);
  else if (nchunks <= 32 * GS_MAX_CHUNKS) gs_split_rows_kernel<GS_MAX_CHUNKS, 32, LIVE><<<mtiles, 256, 0, st>>>(x, ldx, rows, K, im, live);
  else gs_split_rows_wide_kernel<LIVE><<<mtiles * 16, 256, 0, st>>>(x, ldx, rows, K, im, live);
}

extern "C" int rqb200_f32_to_split_image(const float* x, int64_t ldx, int rows, int K, int transposed, void* image, void* stream) {
  RQB_CHECK_ARG(K > 0 && rows >= 0, "f32_to_split_image: bad shape (rows=%d K=%d)", rows, K);
  RQB_CHECK_ARG(transposed ? ldx >= rows : ldx >= K, "f32_to_split_image: ld too small");
  if (rows == 0) return RQB_OK;
  RQB_CHECK_ARG(x && image, "f32_to_split_image: null pointer");
  RQB_CHECK_ARG((reinterpret_cast<uintptr_t>(image) & 15) == 0, "f32_to_split_image: the image must be 16-byte aligned");
  const int mtiles = (rows + 127) / 128;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (transposed) {
    unsigned char* im = reinterpret_cast<unsigned char*>(image);
    const int nkc = (K + GT_KC - 1) / GT_KC;
    if (nkc > 65535) {                                       // grid.y of the column kernels
      rqb_set_error("f32_to_split_image: transposed operand with K = %d > %d", K, 65535 * GT_KC);
      return RQB_ERR_UNSUPPORTED;
    }
    float* scales = reinterpret_cast<float*>(im + 2 * (size_t)mtiles * nkc * GT_BLK_BYTES);
    RQB_CUDA(cudaMemsetAsync(scales, 0, (size_t)mtiles * 128 * sizeof(float), st));
    gs_colmax_kernel<<<dim3((rows + 255) / 256, (K + 127) / 128), 256, 0, st>>>(x, ldx, rows, K, reinterpret_cast<unsigned int*>(scales));
    RQB_LAUNCH_CHECK();
    gs_colscale_kernel<<<(mtiles * 128 + 255) / 256, 256, 0, st>>>(scales, mtiles * 128);
    RQB_LAUNCH_CHECK();
    gs_split_cols_kernel<<<dim3(mtiles, nkc), 256, 0, st>>>(x, ldx, rows, K, im);
  } else {
    gs_split_rows<false>(x, ldx, rows, K, reinterpret_cast<unsigned char*>(image), nullptr, st);
  }
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_f32_to_split_image_counted(const float* x, int64_t ldx, int rows, int K, const int* live_rows, void* image,
                                                 void* stream) {
  RQB_CHECK_ARG(K > 0 && rows >= 0 && ldx >= K, "f32_to_split_image_counted: bad shape (rows=%d K=%d)", rows, K);
  if (rows == 0) return RQB_OK;
  RQB_CHECK_ARG(x && image && live_rows, "f32_to_split_image_counted: null pointer");
  RQB_CHECK_ARG((reinterpret_cast<uintptr_t>(image) & 15) == 0, "f32_to_split_image_counted: the image must be 16-byte aligned");
  gs_split_rows<true>(x, ldx, rows, K, reinterpret_cast<unsigned char*>(image), live_rows, reinterpret_cast<cudaStream_t>(stream));
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

struct GsParams {
  const unsigned char *a_hi, *a_lo, *b_hi, *b_lo;   // [tiles][nkc][16 KB]
  const float *a_scale, *b_scale;                   // 2^-e per image row
  int M, N, nkc, mtiles, nblocks, nitems, relu;
  int ksplit, kc_per;                               // split-K: item = (row tile, column block, k slice of kc_per chunks); slice ks
  int64_t part_stride;                              // writes its partial sums to out + ks * part_stride (ksplit == 1: 0)
  float* out;
  int64_t ldo;
  const float* mask;                                // optional [M, N] (ld = ldm): out = mask > 0 ? out : 0  (ReLU' of a backward GEMM)
  int64_t ldm;
};

// LIVE (rqb200_gemm_split_counted): items are row-tile major, so the live rows' items are the first ones; the others are skipped
// and each live item computes what it computes at the host row count.  The live count is re-read where it is used rather than
// held in a register: the consumers have no register to spare (the host-counted instantiation must stay as it is).
template <bool LIVE>
__device__ __forceinline__ int gs_rows(const GsParams& p, const int* m_live) {
  return LIVE ? min(p.M, max(0, __ldg(m_live))) : p.M;
}
template <bool LIVE>
__device__ __forceinline__ int gs_items(const GsParams& p, const int* m_live) {
  return LIVE ? (gs_rows<LIVE>(p, m_live) + 127) / 128 * p.nblocks * p.ksplit : p.nitems;
}

template <bool LIVE>
__device__ __forceinline__ void gs_gemm(GsParams p, const int* __restrict__ m_live) {
  extern __shared__ __align__(1024) unsigned char gsm[];
  GtSmemMisc* ms = reinterpret_cast<GtSmemMisc*>(gsm + GS_STAGES * GS_STAGE_BYTES);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    if ((smem_u32(gsm) & 1023u) != 0) __trap();
    for (int i = 0; i < GS_STAGES; ++i) { mbar_init(&ms->full[i], 1); mbar_init(&ms->empty[i], 8); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ============================================================== producer: A hi, A lo, B hi, B lo per stage
    if (lane == 0) {
      uint32_t s = 0;
      for (int item = blockIdx.x; item < gs_items<LIVE>(p, m_live); item += gridDim.x) {
        const int ks = item % p.ksplit, tile = item / p.ksplit;
        const int mt = tile / p.nblocks, nbk = tile % p.nblocks;
        const int kc_end = min(p.nkc, (ks + 1) * p.kc_per);
        for (int kc = ks * p.kc_per; kc < kc_end; ++kc, ++s) {
          const uint32_t st = s % GS_STAGES, u = s / GS_STAGES;
          mbar_wait_guarded(&ms->empty[st], (u & 1) ^ 1, 1);
          unsigned char* dst = gsm + st * GS_STAGE_BYTES;
          mbar_expect_tx(&ms->full[st], 4 * GT_BLK_BYTES);
          const size_t ao = ((size_t)mt * p.nkc + kc) * GT_BLK_BYTES, bo = ((size_t)nbk * p.nkc + kc) * GT_BLK_BYTES;
          bulk_g2s(dst, p.a_hi + ao, GT_BLK_BYTES, &ms->full[st]);
          bulk_g2s(dst + GT_BLK_BYTES, p.a_lo + ao, GT_BLK_BYTES, &ms->full[st]);
          bulk_g2s(dst + 2 * GT_BLK_BYTES, p.b_hi + bo, GT_BLK_BYTES, &ms->full[st]);
          bulk_g2s(dst + 3 * GT_BLK_BYTES, p.b_lo + bo, GT_BLK_BYTES, &ms->full[st]);
        }
      }
    }
    return;
  }
  // ============================================================== consumers: hi.hi + lo.hi + hi.lo per k-step
  const int wg = warp >> 2, q4 = lane & 3;
  const int ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const uint32_t base = smem_u32(gsm);
  uint32_t s = 0;
  for (int item = blockIdx.x; item < gs_items<LIVE>(p, m_live); item += gridDim.x) {
    const int ks = item % p.ksplit, tile = item / p.ksplit;
    const int mt = tile / p.nblocks, nbk = tile % p.nblocks;
    const int kc_begin = ks * p.kc_per, kc_end = min(p.nkc, (ks + 1) * p.kc_per);
    // the three products of a 64-wide k chunk accumulate in the tensor core, then the chunk is promoted into an fp32 register
    // total with round-to-nearest adds.  The tensor core truncates its fp32 accumulator after every MMA: summed over the whole
    // K in the tensor core the error grows with the number of MMAs (measured on H100 at K = 512-768: 2-4x that of a plain
    // fp32 GEMM, enough to flip ReLU masks of the MLP backward); promoted every 64 k it stays at the level of a plain fp32 GEMM
    float acc[64], tot[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) tot[i] = 0.f;
    for (int kc = kc_begin; kc < kc_end; ++kc, ++s) {
      const uint32_t st = s % GS_STAGES;
      mbar_wait_guarded(&ms->full[st], (s / GS_STAGES) & 1, 3);
      const uint32_t sa = base + st * GS_STAGE_BYTES + wg * (GT_BLK_BYTES / 2);
      const uint64_t ahi = wg_desc(sa), alo = wg_desc(sa + GT_BLK_BYTES);
      const uint32_t sb = base + st * GS_STAGE_BYTES + 2 * GT_BLK_BYTES;
      const uint64_t bhi = wg_desc(sb), blo = wg_desc(sb + GT_BLK_BYTES);
      wg_fence_acc(acc);
      wg_fence();
#pragma unroll
      for (int j = 0; j < GT_KC / 16; ++j) {
        wg_m64n128_f16(acc, ahi + 2 * j, bhi + 2 * j, j != 0);
        wg_m64n128_f16(acc, alo + 2 * j, bhi + 2 * j, 1);
        wg_m64n128_f16(acc, ahi + 2 * j, blo + 2 * j, 1);
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&ms->empty[st]);
#pragma unroll
      for (int i = 0; i < 64; ++i) tot[i] += acc[i];
    }
    // ---- epilogue: x 2^-(e_row + e_col) -> act -> mask -> fp32 rows.  2^-(e_row + e_col) is applied as two factors of half
    // the exponent each (|e| <= 120 per operand): neither the factor nor the intermediate product leaves the fp32 range
    // unless the result does.  Scale vectors are padded to whole tiles.
    const int col0 = nbk * 128;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = mt * 128 + ra + 8 * h;
      const int ea = (__float_as_int(__ldg(p.a_scale + row)) >> 23) & 0xff;
      float* orow = p.out + (int64_t)ks * p.part_stride + (int64_t)row * p.ldo;
#pragma unroll
      for (int jb = 0; jb < 16; ++jb) {
        const int col = col0 + 8 * jb + 2 * q4;
        if (row >= gs_rows<LIVE>(p, m_live) || col >= p.N) continue;
        const float2 bs = __ldg(reinterpret_cast<const float2*>(p.b_scale + col));
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int et = ea + ((__float_as_int(e ? bs.y : bs.x) >> 23) & 0xff) - 254;     // -(e_row + e_col)
          const int e1 = et >> 1;
          v[e] = (tot[4 * jb + 2 * h + e] * __int_as_float((e1 + 127) << 23)) *
                 __int_as_float((et - e1 + 127) << 23);   // exact
          if (p.relu) v[e] = fmaxf(v[e], 0.f);
          if (p.mask && col + e < p.N && !(__ldg(p.mask + (int64_t)row * p.ldm + col + e) > 0.f)) v[e] = 0.f;
        }
        orow[col] = v[0];
        if (col + 1 < p.N) orow[col + 1] = v[1];
      }
    }
  }
}

__global__ void __launch_bounds__(GT_THREADS, 1) gs_gemm_kernel(GsParams p) { gs_gemm<false>(p, nullptr); }
__global__ void __launch_bounds__(GT_THREADS, 1) gs_gemm_counted_kernel(GsParams p, const int* __restrict__ m_live) {
  gs_gemm<true>(p, m_live);
}

// out[i, j] = sum over the k slices of the partial sums (fixed order: deterministic)
__global__ void gs_reduce_kernel(const float* __restrict__ part, int S, int M, int N, float* __restrict__ out, int64_t ldo) {
  const int64_t n = (int64_t)M * N;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int s = 0; s < S; ++s) acc += part[(int64_t)s * n + i];
    out[(i / N) * ldo + (i % N)] = acc;
  }
}

template <bool LIVE = false>
static int gs_run(const void* a_image, const void* b_image, int M, int N, int K, int relu, const float* mask, int64_t ldm,
                  float* out, int64_t ldo, int ksplit, int kc_per, int64_t part_stride, cudaStream_t st, const int* m_live = nullptr) {
  GsParams p{};
  p.M = M; p.N = N; p.nkc = (K + GT_KC - 1) / GT_KC;
  p.mtiles = (M + 127) / 128;
  p.nblocks = (N + 127) / 128;
  p.ksplit = ksplit; p.kc_per = kc_per; p.part_stride = part_stride;
  p.nitems = p.mtiles * p.nblocks * ksplit;
  p.relu = relu;
  const size_t a_img = (size_t)p.mtiles * p.nkc * GT_BLK_BYTES, b_img = (size_t)p.nblocks * p.nkc * GT_BLK_BYTES;
  p.a_hi = reinterpret_cast<const unsigned char*>(a_image); p.a_lo = p.a_hi + a_img;
  p.a_scale = reinterpret_cast<const float*>(p.a_hi + 2 * a_img);
  p.b_hi = reinterpret_cast<const unsigned char*>(b_image); p.b_lo = p.b_hi + b_img;
  p.b_scale = reinterpret_cast<const float*>(p.b_hi + 2 * b_img);
  p.out = out; p.ldo = ldo;
  p.mask = mask; p.ldm = ldm;
  int dev = 0, sm_count = 0;
  RQB_CUDA(cudaGetDevice(&dev));
  RQB_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
  const size_t smem = (size_t)GS_STAGES * GS_STAGE_BYTES + sizeof(GtSmemMisc);
  const int grid = p.nitems < sm_count ? p.nitems : sm_count;
  if (LIVE) {
    RQB_CUDA(cudaFuncSetAttribute(gs_gemm_counted_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gs_gemm_counted_kernel<<<grid, GT_THREADS, smem, st>>>(p, m_live);
  } else {
    RQB_CUDA(cudaFuncSetAttribute(gs_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gs_gemm_kernel<<<grid, GT_THREADS, smem, st>>>(p);
  }
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_gemm_split(const void* a_image, const void* b_image, int M, int N, int K, int relu, const float* mask,
                                 int64_t ldm, float* out, int64_t ldo, void* stream) {
  RQB_CHECK_ARG(M >= 0 && N > 0 && K > 0 && ldo >= N, "gemm_split: bad shape (M=%d N=%d K=%d ldo=%lld)", M, N, K, (long long)ldo);
  if (M == 0) return RQB_OK;
  RQB_CHECK_ARG(a_image && b_image && out, "gemm_split: null pointer");
  RQB_CHECK_ARG(!mask || ldm >= N, "gemm_split: ldm < N");
  return gs_run(a_image, b_image, M, N, K, relu, mask, ldm, out, ldo, 1, (K + GT_KC - 1) / GT_KC, 0,
                reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int rqb200_gemm_split_counted(const void* a_image, const void* b_image, int M, int N, int K, int relu, const float* mask,
                                         int64_t ldm, const int* live_m, float* out, int64_t ldo, void* stream) {
  RQB_CHECK_ARG(M >= 0 && N > 0 && K > 0 && ldo >= N, "gemm_split_counted: bad shape (M=%d N=%d K=%d ldo=%lld)", M, N, K,
                (long long)ldo);
  if (M == 0) return RQB_OK;
  RQB_CHECK_ARG(a_image && b_image && out && live_m, "gemm_split_counted: null pointer");
  RQB_CHECK_ARG(!mask || ldm >= N, "gemm_split_counted: ldm < N");
  return gs_run<true>(a_image, b_image, M, N, K, relu, mask, ldm, out, ldo, 1, (K + GT_KC - 1) / GT_KC, 0,
                      reinterpret_cast<cudaStream_t>(stream), live_m);
}

// Split-K schedule for products with few output tiles and a long contraction (the weight gradients: M = out, N = in, K = batch):
// the k chunks are cut into `slices` ranges, every (tile, range) is a work item writing partial sums into the workspace
// [slices][M][N], and a fixed-order reduction produces out.  gemm_split_k_slices picks the slice count that fills the SMs.
extern "C" int rqb200_gemm_split_k_slices(int M, int N, int K) {
  if (M <= 0 || N <= 0 || K <= 0) return 1;
  int dev = 0, sm_count = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
  const int nkc = (K + GT_KC - 1) / GT_KC;
  const int tiles = ((M + 127) / 128) * ((N + 127) / 128);
  int want = (sm_count + tiles - 1) / tiles;                 // slices that give every SM an item
  if (want > nkc / 4) want = nkc / 4;                        // at least 4 chunks (256 k) per slice
  if (want < 1) want = 1;
  const int kc_per = (nkc + want - 1) / want;
  return (nkc + kc_per - 1) / kc_per;                        // no empty slice
}

extern "C" int rqb200_gemm_split_k(const void* a_image, const void* b_image, int M, int N, int K, int slices, float* workspace,
                                   float* out, int64_t ldo, void* stream) {
  RQB_CHECK_ARG(M >= 0 && N > 0 && K > 0 && ldo >= N && slices >= 1, "gemm_split_k: bad shape (M=%d N=%d K=%d slices=%d)", M, N, K, slices);
  if (M == 0) return RQB_OK;
  RQB_CHECK_ARG(a_image && b_image && out, "gemm_split_k: null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int nkc = (K + GT_KC - 1) / GT_KC;
  const int kc_per = (nkc + slices - 1) / slices;
  RQB_CHECK_ARG((int64_t)(slices - 1) * kc_per < nkc, "gemm_split_k: %d slices of %d chunks leave an empty slice (K = %d)", slices, kc_per, K);
  if (slices == 1) return gs_run(a_image, b_image, M, N, K, 0, nullptr, 0, out, ldo, 1, nkc, 0, st);
  RQB_CHECK_ARG(workspace, "gemm_split_k: null workspace");
  int rc = gs_run(a_image, b_image, M, N, K, 0, nullptr, 0, workspace, N, slices, kc_per, (int64_t)M * N, st);
  if (rc) return rc;
  const int64_t n = (int64_t)M * N;
  int grid = (int)((n + 255) / 256);
  if (grid > 132 * 8) grid = 132 * 8;
  gs_reduce_kernel<<<grid, 256, 0, st>>>(workspace, slices, M, N, out, ldo);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}
