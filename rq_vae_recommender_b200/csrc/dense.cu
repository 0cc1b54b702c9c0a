// Exact-fp32 dense helpers around the quantiser: strided SGEMM with fused ReLU / mask epilogues (the encoder and
// decoder MLPs of modules/encoder.py and the W@C / grad GEMMs of the Gumbel-softmax path), the Gumbel-softmax
// row kernels (distributions/gumbel.py + modules/quantize.py:131-136), distance rows, row L2 normalisation.
#include "common.cuh"
#include <cmath>

// ------------------------------------------------------------------------------------------------ SGEMM
// C[m,n] = epi( alpha * sum_k A(m,k) B(k,n) + beta * C[m,n] ),  A(m,k) = A[m*sAm + k*sAk], B(k,n) = B[k*sBk + n*sBn]
// epi: relu -> max(0, .);  mask -> multiply by (mask[m,n] > 0)   (ReLU backward)
#define SG_BM 128
#define SG_BN 128
#define SG_BK 16
#define SG_THREADS 256

struct SgemmParams {
  const float* A; int64_t sAm, sAk;
  const float* B; int64_t sBk, sBn;
  float* C; int64_t ldc;
  const float* mask; int64_t ldmask;
  int M, N, K;
  float alpha, beta;
  int relu;
};

__global__ void __launch_bounds__(SG_THREADS) sgemm_kernel(SgemmParams p) {
  __shared__ __align__(16) float As[2][SG_BK][SG_BM + 4];
  __shared__ __align__(16) float Bs[2][SG_BK][SG_BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * SG_BM, n0 = blockIdx.x * SG_BN;
  const int ty = tid >> 4, tx = tid & 15;  // 16 x 16 threads, 8 x 8 outputs each

  // loader mappings: walk the unit-stride dimension with consecutive threads
  const bool a_k_fast = (p.sAk == 1);
  const bool b_n_fast = (p.sBn == 1);

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float ra[8], rb[8];
  auto gload = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int e = tid + i * SG_THREADS;  // 0 .. 2047
      int m, k;
      if (a_k_fast) { k = e & (SG_BK - 1); m = e >> 4; } else { m = e & (SG_BM - 1); k = e >> 7; }
      const int gm = m0 + m, gk = k0 + k;
      ra[i] = (gm < p.M && gk < p.K) ? __ldg(p.A + gm * p.sAm + gk * p.sAk) : 0.f;
      int n, kb;
      if (b_n_fast) { n = e & (SG_BN - 1); kb = e >> 7; } else { kb = e & (SG_BK - 1); n = e >> 4; }
      const int gn = n0 + n, gkb = k0 + kb;
      rb[i] = (gn < p.N && gkb < p.K) ? __ldg(p.B + gkb * p.sBk + gn * p.sBn) : 0.f;
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int e = tid + i * SG_THREADS;
      int m, k;
      if (a_k_fast) { k = e & (SG_BK - 1); m = e >> 4; } else { m = e & (SG_BM - 1); k = e >> 7; }
      As[buf][k][m] = ra[i];
      int n, kb;
      if (b_n_fast) { n = e & (SG_BN - 1); kb = e >> 7; } else { kb = e & (SG_BK - 1); n = e >> 4; }
      Bs[buf][kb][n] = rb[i];
    }
  };

  const int nk = (p.K + SG_BK - 1) / SG_BK;
  gload(0);
  sstore(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) gload((kt + 1) * SG_BK);
#pragma unroll
    for (int k = 0; k < SG_BK; ++k) {
      float a[8], b[8];
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      sstore(buf ^ 1);
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (gm >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int gn = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (gn >= p.N) continue;
      float v = p.alpha * acc[i][j];
      float* c = p.C + (int64_t)gm * p.ldc + gn;
      if (p.beta != 0.f) v += p.beta * *c;
      if (p.relu) v = fmaxf(v, 0.f);
      if (p.mask && !(__ldg(p.mask + (int64_t)gm * p.ldmask + gn) > 0.f)) v = 0.f;
      *c = v;
    }
  }
}

extern "C" int rqb200_sgemm(int transA, int transB, int M, int N, int K, float alpha, const float* A, int64_t lda,
                            const float* B, int64_t ldb, float beta, float* C, int64_t ldc, int relu,
                            const float* mask, int64_t ldmask, void* stream) {
  RQB_CHECK_ARG(M >= 0 && N >= 0 && K >= 0, "sgemm: negative dimension");
  if (M == 0 || N == 0) return RQB_OK;
  RQB_CHECK_ARG(A && B && C, "sgemm: null pointer");
  SgemmParams p;
  p.A = A; p.B = B; p.C = C; p.ldc = ldc; p.mask = mask; p.ldmask = ldmask;
  p.M = M; p.N = N; p.K = K; p.alpha = alpha; p.beta = beta; p.relu = relu;
  // row-major storage: A is [M,K] (or [K,M] if transA), B is [K,N] (or [N,K] if transB)
  if (transA) { p.sAm = 1; p.sAk = lda; } else { p.sAm = lda; p.sAk = 1; }
  if (transB) { p.sBk = 1; p.sBn = ldb; } else { p.sBk = ldb; p.sBn = 1; }
  dim3 grid((N + SG_BN - 1) / SG_BN, (M + SG_BM - 1) / SG_BM);
  sgemm_kernel<<<grid, SG_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ------------------------------------------------------------------------------------------------ row kernels
// dist[b,k] = (||x_b||^2 + ||c_k||^2) - 2 dot[b,k]  in place on a [B,K] buffer of dots (quantize.py:113-117),
// plus first-index argmin per row (quantize.py:128).  One warp per row.
__global__ void dist_finish_kernel(float* dots, const float* x, int64_t ldx, const float* cc, int B, int D, int K,
                                   int64_t* ids) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= B) return;
  float s = 0.f;
  for (int d = lane; d < D; d += 32) { const float v = __ldg(x + (int64_t)row * ldx + d); s = fmaf(v, v, s); }
  s = warp_sum(s);
  float bv = INFINITY; int bi = 0x7fffffff;
  for (int k = lane; k < K; k += 32) {
    const float dist = (s + __ldg(cc + k)) - 2.f * dots[(int64_t)row * K + k];
    dots[(int64_t)row * K + k] = dist;
    if (dist < bv) { bv = dist; bi = k; }
  }
  warp_argmin(bv, bi);
  if (lane == 0 && ids) ids[row] = bi < K ? bi : 0;
}

__global__ void row_sqnorm_kernel(const float* c, int K, int D, float* out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= K) return;
  float s = 0.f;
  for (int d = lane; d < D; d += 32) { const float v = c[(int64_t)row * D + d]; s = fmaf(v, v, s); }
  s = warp_sum(s);
  if (lane == 0) out[row] = s;
}

// W = softmax((-dist + G)/T), G = -log(-log(U+eps)+eps)    (gumbel.py:8-20, quantize.py:132-134)
__global__ void gumbel_softmax_fwd_kernel(const float* dist, const float* u, float* w, int B, int K, float inv_t_dummy,
                                          float temperature) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= B) return;
  const float* dr = dist + (int64_t)row * K;
  const float* ur = u + (int64_t)row * K;
  float* wr = w + (int64_t)row * K;
  float mx = -INFINITY;
  for (int k = lane; k < K; k += 32) {
    const float g = -logf(-logf(ur[k] + 1e-20f) + 1e-20f);
    const float y = (-dr[k] + g) / temperature;
    wr[k] = y;
    mx = fmaxf(mx, y);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int k = lane; k < K; k += 32) { const float e = expf(wr[k] - mx); wr[k] = e; sum += e; }
  sum = warp_sum(sum);
  for (int k = lane; k < K; k += 32) wr[k] = wr[k] / sum;
}

// per row: loss = ||x-E||^2 + beta ||x-E||^2 ; res_next = x - E ; ||E||     (loss.py:38-41, rqvae.py:130,158)
__global__ void gumbel_row_finish_kernel(const float* x, int64_t ldx, const float* E, int B, int D, float beta,
                                         float* loss) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= B) return;
  float s = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float df = __ldg(x + (int64_t)row * ldx + d) - E[(int64_t)row * D + d];
    s = fmaf(df, df, s);
  }
  s = warp_sum(s);
  if (lane == 0) loss[row] = s + beta * s;
}

// gE = g_out + 2 gamma (E - x)
__global__ void gumbel_bwd_ge_kernel(const float* g_out, int64_t go_sB, int64_t go_sD, const float* g_loss,
                                     int64_t gl_sB, const float* x, int64_t ldx, const float* E, float* gE, int B,
                                     int D) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * D) return;
  const int row = (int)(i / D), d = (int)(i % D);
  const float go = g_out ? g_out[row * go_sB + d * go_sD] : 0.f;
  const float gm = g_loss ? g_loss[row * gl_sB] : 0.f;
  gE[i] = go + 2.f * gm * (E[i] - x[(int64_t)row * ldx + d]);
}

// gdist = -W * (gW - sum_k W gW) / T  (in place over gW);  rowsum[b] = sum_k gdist ; colsum[k] += gdist
// Column sums: every CTA walks its rows (grid-stride) and keeps the K partial sums in shared memory, one global atomic per column
// and CTA at the end (one atomic per ELEMENT into 256 addresses ran at 3 % of the SM throughput)
__global__ void gumbel_bwd_softmax_kernel(const float* w, float* gw, int B, int K, float temperature, float* rowsum,
                                          float* colsum) {
  extern __shared__ float s_col[];                            // [K] (K <= GUMBEL_SMEM_K), else straight to global
  const bool use_s = K <= 8192;
  if (use_s)
    for (int k = threadIdx.x; k < K; k += blockDim.x) s_col[k] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < B; row += gridDim.x * wpb) {
    const float* wr = w + (int64_t)row * K;
    float* gr = gw + (int64_t)row * K;
    float dot = 0.f;
    for (int k = lane; k < K; k += 32) dot = fmaf(wr[k], gr[k], dot);
    dot = warp_sum(dot);
    float rs = 0.f;
    for (int k = lane; k < K; k += 32) {
      const float gd = -(wr[k] * (gr[k] - dot) / temperature);
      gr[k] = gd;
      rs += gd;
      atomicAdd(use_s ? s_col + k : colsum + k, gd);
    }
    rs = warp_sum(rs);
    if (lane == 0) rowsum[row] = rs;
  }
  __syncthreads();
  if (use_s)
    for (int k = threadIdx.x; k < K; k += blockDim.x) atomicAdd(colsum + k, s_col[k]);
}

// gx = 2 beta gamma (x - E) + 2 x rowsum - 2 (gdist @ C)   where `acc` holds gdist @ C on entry   [B,D]
__global__ void gumbel_bwd_gx_kernel(float* acc, const float* x, int64_t ldx, const float* E, const float* g_loss,
                                     int64_t gl_sB, const float* rowsum, float beta, int B, int D) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * D) return;
  const int row = (int)(i / D), d = (int)(i % D);
  const float xv = x[(int64_t)row * ldx + d];
  const float gm = g_loss ? g_loss[row * gl_sB] : 0.f;
  acc[i] = 2.f * beta * gm * (xv - E[i]) + 2.f * xv * rowsum[row] - 2.f * acc[i];
}

// gC += 2 C colsum[k]   (the (c^2).sum term of dist)    [K,D]
__global__ void gumbel_bwd_gc_kernel(float* gC, const float* C, const float* colsum, int K, int D) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * D) return;
  gC[i] += 2.f * C[i] * colsum[i / D];
}

// y = x / max(||x||, eps) per row (modules/normalize.py:6-7); norms kept for the backward
__global__ void l2norm_fwd_kernel(const float* x, float* y, float* norms, int B, int D, float eps) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= B) return;
  float s = 0.f;
  for (int d = lane; d < D; d += 32) { const float v = x[(int64_t)row * D + d]; s = fmaf(v, v, s); }
  const float n = sqrtf(warp_sum(s));
  const float den = fmaxf(n, eps);
  for (int d = lane; d < D; d += 32) y[(int64_t)row * D + d] = x[(int64_t)row * D + d] / den;
  if (lane == 0 && norms) norms[row] = n;
}

// gx = (gy - y (gy.y)) / max(n, eps)   [for n > eps; for n <= eps the clamp is constant: gx = gy/eps]
__global__ void l2norm_bwd_kernel(const float* gy, const float* y, const float* norms, float* gx, int B, int D,
                                  float eps) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= B) return;
  const float n = norms[row];
  float dot = 0.f;
  for (int d = lane; d < D; d += 32) dot = fmaf(gy[(int64_t)row * D + d], y[(int64_t)row * D + d], dot);
  dot = warp_sum(dot);
  if (!(n > eps)) dot = 0.f;
  const float den = fmaxf(n, eps);
  for (int d = lane; d < D; d += 32)
    gx[(int64_t)row * D + d] = (gy[(int64_t)row * D + d] - y[(int64_t)row * D + d] * dot) / den;
}

#define ROW_GRID(B) (((B) + 7) / 8), 256
#define ELT_GRID(n) (unsigned)(((n) + 255) / 256), 256

extern "C" int rqb200_row_sqnorm(const float* c, int K, int D, float* out, void* stream) {
  if (K == 0) return RQB_OK;
  RQB_CHECK_ARG(c && out, "row_sqnorm: null pointer");
  row_sqnorm_kernel<<<ROW_GRID(K), 0, reinterpret_cast<cudaStream_t>(stream)>>>(c, K, D, out);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_dist_finish(float* dots, const float* x, int64_t ldx, const float* cc, int B, int D, int K,
                                  int64_t* ids, void* stream) {
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(dots && x && cc, "dist_finish: null pointer");
  dist_finish_kernel<<<ROW_GRID(B), 0, reinterpret_cast<cudaStream_t>(stream)>>>(dots, x, ldx, cc, B, D, K, ids);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_gumbel_softmax_fwd(const float* dist, const float* uniform, float* weights, int B, int K,
                                         float temperature, void* stream) {
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(dist && uniform && weights && temperature > 0.f, "gumbel_softmax_fwd: bad argument");
  gumbel_softmax_fwd_kernel<<<ROW_GRID(B), 0, reinterpret_cast<cudaStream_t>(stream)>>>(dist, uniform, weights, B, K,
                                                                                       0.f, temperature);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_gumbel_row_finish(const float* x, int64_t ldx, const float* E, int B, int D, float beta,
                                        float* loss, void* stream) {
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(x && E && loss, "gumbel_row_finish: null pointer");
  gumbel_row_finish_kernel<<<ROW_GRID(B), 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, ldx, E, B, D, beta, loss);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_gumbel_bwd_ge(const float* g_out, int64_t go_sB, int64_t go_sD, const float* g_loss,
                                    int64_t gl_sB, const float* x, int64_t ldx, const float* E, float* gE, int B, int D,
                                    void* stream) {
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(x && E && gE, "gumbel_bwd_ge: null pointer");
  gumbel_bwd_ge_kernel<<<ELT_GRID((int64_t)B * D), 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      g_out, go_sB, go_sD, g_loss, gl_sB, x, ldx, E, gE, B, D);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_gumbel_bwd_softmax(const float* weights, float* gw_inout, int B, int K, float temperature,
                                         float* rowsum, float* colsum, void* stream) {
  RQB_CHECK_ARG(weights && gw_inout && rowsum && colsum, "gumbel_bwd_softmax: null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RQB_CUDA(cudaMemsetAsync(colsum, 0, (size_t)K * sizeof(float), st));
  if (B == 0) return RQB_OK;
  int grid = (B + 7) / 8;
  if (grid > 132 * 4) grid = 132 * 4;
  gumbel_bwd_softmax_kernel<<<grid, 256, K <= 8192 ? (size_t)K * sizeof(float) : 0, st>>>(weights, gw_inout, B, K, temperature, rowsum, colsum);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_gumbel_bwd_gx(float* acc_inout, const float* x, int64_t ldx, const float* E, const float* g_loss,
                                    int64_t gl_sB, const float* rowsum, float beta, int B, int D, void* stream) {
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(acc_inout && x && E && rowsum, "gumbel_bwd_gx: null pointer");
  gumbel_bwd_gx_kernel<<<ELT_GRID((int64_t)B * D), 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      acc_inout, x, ldx, E, g_loss, gl_sB, rowsum, beta, B, D);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_gumbel_bwd_gc(float* gC_inout, const float* C, const float* colsum, int K, int D, void* stream) {
  RQB_CHECK_ARG(gC_inout && C && colsum, "gumbel_bwd_gc: null pointer");
  gumbel_bwd_gc_kernel<<<ELT_GRID((int64_t)K * D), 0, reinterpret_cast<cudaStream_t>(stream)>>>(gC_inout, C, colsum, K, D);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_l2norm_fwd(const float* x, float* y, float* norms, int B, int D, float eps, void* stream) {
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(x && y, "l2norm_fwd: null pointer");
  l2norm_fwd_kernel<<<ROW_GRID(B), 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, y, norms, B, D, eps);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_l2norm_bwd(const float* gy, const float* y, const float* norms, float* gx, int B, int D,
                                 float eps, void* stream) {
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(gy && y && norms && gx, "l2norm_bwd: null pointer");
  l2norm_bwd_kernel<<<ROW_GRID(B), 0, reinterpret_cast<cudaStream_t>(stream)>>>(gy, y, norms, gx, B, D, eps);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ------------------------------------------------------------------------------------------------ id statistics
// per-level code usage histogram (train_rqvae.py:285-289): shared-memory bins, one global atomic per bin per block
__global__ void sid_histogram_kernel(const int64_t* ids, int B, int L, int K, unsigned long long* hist) {
  extern __shared__ unsigned int bins[];  // [L*K]
  for (int i = threadIdx.x; i < L * K; i += blockDim.x) bins[i] = 0;
  __syncthreads();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (int64_t)B * L; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = (int)(i % L);
    const int64_t v = ids[i];
    if (v >= 0 && v < K) atomicAdd(&bins[l * K + (int)v], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < L * K; i += blockDim.x)
    if (bins[i]) atomicAdd(hist + i, (unsigned long long)bins[i]);
}

extern "C" int rqb200_sid_histogram(const int64_t* ids, int B, int L, int K, int64_t* hist, void* stream) {
  RQB_CHECK_ARG(hist && L > 0 && K > 0 && (size_t)L * K * 4 <= 160 * 1024, "sid_histogram: bad argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RQB_CUDA(cudaMemsetAsync(hist, 0, (size_t)L * K * sizeof(int64_t), st));
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(ids, "sid_histogram: null ids");
  const size_t smem = (size_t)L * K * sizeof(unsigned int);
  if (smem > 48 * 1024)
    RQB_CUDA(cudaFuncSetAttribute(sid_histogram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = (int)(((int64_t)B * L + 255) / 256);
  if (grid > 132 * 4) grid = 132 * 4;
  sid_histogram_kernel<<<grid, 256, smem, st>>>(ids, B, L, K, reinterpret_cast<unsigned long long*>(hist));
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}
