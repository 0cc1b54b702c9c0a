// Tensor-core tokeniser for sm_90a: prepared codebook state + C-ABI entry points (the kernels are in csrc/rq_tcx.cu).
//
// Result contract: identical to rqb200_rq_forward(mode = EVAL, ids only) -- the hard-argmin chain of
// modules/quantize.py:113-128,159-161 x L + modules/rqvae.py:125-132 (what semids.py:125 consumes).
//
// Why tensor cores: the distance term x.c^T is 2*D*K*L = 1.18 MFLOP per 3 KB item (381 FLOP/B, SURVEY 8d);
// on CUDA cores the pass is ~30x compute bound.  Why it is still exact: the fp16 product only FILTERS.
//   S_l[b,k]  = fp16(x_b) . fp16(c_{l,k})            (wgmma, fp32 accumulate in registers; exact power-of-two scales)
//   score_l   = cc_{l,k} - 2 (S_l - sum_{j<l} G_{jl}[id_j, k])     (G = fp32 Gram tables C_j C_l^T, so every level is
//               scored from the ONE fp16 image of x: the residual never has to be re-quantised or re-staged)
//   candidates = { k : score <= min + 4 eps_b }      eps_b bounds the fp16 rounding of the dot product (margin in the epilogue)
//   |candidates| == 1  -> that code is the exact argmin;  else the candidates are re-scored with the exact fp32
//   arithmetic of the CUDA-core kernel (sequential fp32 residual, (xx + cc) - 2 dot, first index wins ties).
//
// K = 256 m codes per level, m = 1..8.  The Gram tables cost K^2 L(L-1)/2 x 4 bytes of state (50 MB at K = 2048, L = 3;
// 470 MB at L = 8) and l K 4 bytes of reads per row at level l; prepare computes them in float64, (K / 16)^2 blocks per table.
//
#include "tc_common.cuh"

int tcx_run(const float* x, int64_t ldx, int B, const void* state, int D, int K, int L, int64_t* ids, int* stats, int sm_count,
            cudaStream_t st);
int tcx_ring_stages(int D, int K, int L);

extern "C" int rqb200_tokenize_tc_supported(int D, int K, int L) {
  return (K >= TC_K && K <= TC_MAX_K && K % TC_K == 0 && D >= TC_KC && D <= TC_MAX_D && D % TC_KC == 0 && L >= 1 &&
          L <= RQB_MAX_LEVELS) ? 1 : 0;
}

extern "C" size_t rqb200_tokenize_tc_state_bytes(int D, int K, int L) {
  if (!rqb200_tokenize_tc_supported(D, K, L)) return 0;
  return tc_state_size(D, K, L);
}

extern "C" int rqb200_tokenize_tc_ring_stages(int D, int K, int L) {
  if (!rqb200_tokenize_tc_supported(D, K, L)) return 0;
  return tcx_ring_stages(D, K, L);
}

// ------------------------------------------------------------------------------------------------ prepare
// cbptr[l]: level l of the state's fp32 codebook copy
__global__ void tc_prep_ptrs_kernel(const float** cbptr, const float* cbf, size_t level_elems, int L) {
  if (threadIdx.x < L) cbptr[threadIdx.x] = cbf + threadIdx.x * level_elems;
}

// hcc[l][k] = cc/2 from a float64 sum (the filter's table); amax and c2max of the level
__global__ void tc_prep_stats_kernel(const float* const* cbs, int D, int K, TcHeader* hdr, float* hcc) {
  const int l = blockIdx.y;
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= K) return;
  const float* c = cbs[l] + (int64_t)k * D;
  double s2 = 0.0;
  float mx = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float v = c[d];
    s2 += (double)v * (double)v;
    mx = fmaxf(mx, fabsf(v));
  }
  s2 = warp_sum_d(s2);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) {
    hcc[l * K + k] = (float)(0.5 * s2);
    atomicMax(&hdr->amax_bits[l], __float_as_uint(mx));
    atomicMax(&hdr->c2_bits[l], __float_as_uint(__double2float_ru(sqrt(s2))));
  }
}

// cc[l][k] = sum_d c^2 in fp32, lane-strided fma + shuffle tree: bit-identical to rq_prep_norm_kernel (csrc/rq_simt.cu), it is
// the value the exact re-rank adds in (xx + cc) - 2 dot
__global__ void tc_prep_cc_kernel(const float* const* cbs, int D, int K, float* cc) {
  const int l = blockIdx.y;
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= K) return;
  const float* c = cbs[l] + (int64_t)k * D;
  float s2 = 0.f;
  for (int d = lane; d < D; d += 32) s2 = fmaf(c[d], c[d], s2);
  s2 = warp_sum(s2);
  if (lane == 0) cc[l * K + k] = s2;
}

__global__ void tc_prep_scale_kernel(TcHeader* hdr, int L) {
  const int l = threadIdx.x;
  if (l >= L) return;
  const float amax = __uint_as_float(hdr->amax_bits[l]);
  float sc = 1.f;
  if (amax > 0.f && isfinite(amax)) {
    int e;
    frexpf(amax, &e);          // amax = m * 2^e, m in [0.5, 1)
    e = max(-60, min(60, e));
    sc = ldexpf(1.f, -e);      // amax * sc in [0.5, 1)
  }
  hdr->lv[l].sc = sc;
}

// measured fp16 rounding of every code: chat = max_k ||c~_k||, ec = max_k ||c~_k - c_k||  (c~ = fp16(c sc) / sc), float64 sums
__global__ void tc_prep_err_kernel(const float* const* cbs, int D, int K, TcHeader* hdr) {
  const int l = blockIdx.y;
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= K) return;
  const float sc = hdr->lv[l].sc;
  const double inv = 1.0 / (double)sc;
  const float* c = cbs[l] + (int64_t)k * D;
  double n2 = 0.0, e2 = 0.0;
  for (int d = lane; d < D; d += 32) {
    const double v = (double)c[d];
    const double t = (double)__half2float(__float2half_rn(c[d] * sc)) * inv;
    n2 += t * t;
    e2 += (t - v) * (t - v);
  }
  n2 = warp_sum_d(n2); e2 = warp_sum_d(e2);
  if (lane == 0) {   // non-negative floats order like their bit patterns; inf / NaN sort above every finite value
    atomicMax(&hdr->chat_bits[l], __float_as_uint(__double2float_ru(sqrt(n2))));
    atomicMax(&hdr->ec_bits[l], __float_as_uint(__double2float_ru(sqrt(e2))));
  }
}

__global__ void tc_prep_consts_kernel(TcHeader* hdr, int L) {
  const int l = threadIdx.x;
  if (l >= L) return;
  TcLevelConst& c = hdr->lv[l];
  c.chat = TC_INFL * __uint_as_float(hdr->chat_bits[l]);
  c.ec = TC_INFL * __uint_as_float(hdr->ec_bits[l]);
  c.c2max = __uint_as_float(hdr->c2_bits[l]);
  float g = 0.f;
  for (int j = 0; j < l; ++j) g += __uint_as_float(hdr->c2_bits[j]);
  c.prior = g;
  c.gerr = 2.38418579e-7f * (c.c2max * g + 0.5f * c.c2max * c.c2max);   // 2^-22: tables from float64 rounded once, <= 4 fp32 roundings after
}

// Bblob[(l*(K/128)+h)*nkc + kc] = 16 KB smem image of codes [128h, 128h+128) x k [64kc, 64kc+64):
// K-major, 128 B per code row, 16-byte chunks XOR-swizzled with (row & 7)  (the wgmma SWIZZLE_128B canonical layout); the blocks
// h = 2nb and h = 2nb + 1 of a (level, chunk) form the 256-code operand of code block nb in shared memory
__global__ void tc_prep_blob_kernel(const float* const* cbs, int D, int K, const TcHeader* hdr, __half* blob) {
  const int nkc = D / TC_KC, nh = K / 128;
  const int blk = blockIdx.x;  // (l*nh+h)*nkc + kc
  const int kc = blk % nkc, h = (blk / nkc) % nh, l = blk / (nh * nkc);
  const float sc = hdr->lv[l].sc;
  const float* c = cbs[l];
  __half* out = blob + (size_t)blk * (TC_BSTAGE_BYTES / 2);
  for (int i = threadIdx.x; i < 128 * TC_KC; i += blockDim.x) {
    const int n = i / TC_KC, k = i % TC_KC;
    const float v = c[(int64_t)(h * 128 + n) * D + kc * TC_KC + k] * sc;
    const int chunk = (k >> 3) ^ (n & 7);
    out[n * 64 + chunk * 8 + (k & 7)] = __float2half_rn(v);
  }
}

// Gram table G_{j,l}[i][k] = c_{j,i} . c_{l,k} accumulated in float64 and rounded to fp32 ONCE; for j = 0 the level's cc_l[k] / 2 is
// folded in before the rounding, so the epilogue scores with one table sum:  h[k] = T[k] - S[k] / sc,
// T = cc/2 + sum_j G_{j,l}[id_j]  (argmin-equivalent to quantize.py:113-117).  16 x 16 outputs per block, k tiles of 16 through smem.
__global__ void __launch_bounds__(256) tc_prep_gram_kernel(const float* __restrict__ cj, const float* __restrict__ cl, int D,
                                                           int K, float* __restrict__ g, int fold_cc) {
  __shared__ float sa[16][17], sb[16][17];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int i = blockIdx.y * 16 + ty, k = blockIdx.x * 16 + tx;
  double acc = 0.0, cck = 0.0;
  for (int d0 = 0; d0 < D; d0 += 16) {
    sa[ty][tx] = cj[(int64_t)(blockIdx.y * 16 + ty) * D + d0 + tx];
    sb[ty][tx] = cl[(int64_t)(blockIdx.x * 16 + ty) * D + d0 + tx];
    __syncthreads();
#pragma unroll
    for (int d = 0; d < 16; ++d) {
      const double b = (double)sb[tx][d];
      acc += (double)sa[ty][d] * b;
      cck += b * b;
    }
    __syncthreads();
  }
  g[(size_t)i * K + k] = (float)(fold_cc ? acc + 0.5 * cck : acc);
}

extern "C" int rqb200_tokenize_tc_prepare(const float* const* codebooks, int D, int K, int L, void* state,
                                          size_t state_bytes, void* stream) {
  if (!rqb200_tokenize_tc_supported(D, K, L)) {
    rqb_set_error("tokenize_tc: shape D=%d K=%d L=%d not supported (need K = 256 m with 1 <= m <= 8, D %% 64 == 0, 64 <= D <= 768)", D, K, L);
    return RQB_ERR_UNSUPPORTED;
  }
  RQB_CHECK_ARG(codebooks && state, "tokenize_tc_prepare: null pointer");
  if (state_bytes < rqb200_tokenize_tc_state_bytes(D, K, L)) {
    rqb_set_error("tokenize_tc_prepare: state too small");
    return RQB_ERR_WORKSPACE;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  char* base = reinterpret_cast<char*>(state);
  TcHeader* hdr = reinterpret_cast<TcHeader*>(base);
  float* cc = reinterpret_cast<float*>(base + tc_off_cc(K, L));
  float* hcc = reinterpret_cast<float*>(base + tc_off_hcc(K, L));
  float* gram = reinterpret_cast<float*>(base + tc_off_gram(K, L));
  const float** cbptr = reinterpret_cast<const float**>(base + tc_off_cbptr(K, L));
  __half* blob = reinterpret_cast<__half*>(base + tc_off_blob(D, K, L));
  float* cbf = reinterpret_cast<float*>(base + tc_off_cbf(K, L));
  RQB_CUDA(cudaMemsetAsync(hdr, 0, sizeof(TcHeader), st));
  // fp32 copy for the exact re-rank: 256-byte aligned rows whatever the caller's tensors look like, and the prepared state
  // no longer references caller memory after this call returns (stream order); every prepare kernel reads the copy
  for (int l = 0; l < L; ++l)
    RQB_CUDA(cudaMemcpyAsync(cbf + (size_t)l * K * D, codebooks[l], sizeof(float) * K * D, cudaMemcpyDeviceToDevice, st));
  // the level pointer table is written on the device: a copy from pageable host memory may wait for the stream's earlier work,
  // and the prepare must never block the host
  tc_prep_ptrs_kernel<<<1, 32, 0, st>>>(cbptr, cbf, (size_t)K * D, L);
  RQB_LAUNCH_CHECK();
  tc_prep_stats_kernel<<<dim3(K / 8, L), 256, 0, st>>>(cbptr, D, K, hdr, hcc);
  RQB_LAUNCH_CHECK();
  tc_prep_cc_kernel<<<dim3(K / 8, L), 256, 0, st>>>(cbptr, D, K, cc);
  RQB_LAUNCH_CHECK();
  tc_prep_scale_kernel<<<1, 32, 0, st>>>(hdr, L);
  RQB_LAUNCH_CHECK();
  tc_prep_err_kernel<<<dim3(K / 8, L), 256, 0, st>>>(cbptr, D, K, hdr);
  RQB_LAUNCH_CHECK();
  tc_prep_consts_kernel<<<1, 32, 0, st>>>(hdr, L);
  RQB_LAUNCH_CHECK();
  tc_prep_blob_kernel<<<L * (K / 128) * (D / TC_KC), 256, 0, st>>>(cbptr, D, K, hdr, blob);
  RQB_LAUNCH_CHECK();
  for (int l = 1; l < L; ++l)
    for (int j = 0; j < l; ++j) {
      float* g = gram + (size_t)(l * (l - 1) / 2 + j) * K * K;
      tc_prep_gram_kernel<<<dim3(K / 16, K / 16), 256, 0, st>>>(cbf + (size_t)j * K * D, cbf + (size_t)l * K * D, D, K, g, j == 0);
      RQB_LAUNCH_CHECK();
    }
  return RQB_OK;
}


extern "C" int rqb200_tokenize_tc_run(const float* x, int64_t ldx, int B, const void* state, int D, int K, int L,
                                      int64_t* ids, int* stats, void* stream) {
  if (!rqb200_tokenize_tc_supported(D, K, L)) {
    rqb_set_error("tokenize_tc: shape D=%d K=%d L=%d not supported", D, K, L);
    return RQB_ERR_UNSUPPORTED;
  }
  RQB_CHECK_ARG(B >= 0 && ldx >= D && ldx < (1 << 24), "tokenize_tc_run: bad shape");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(x && state && ids, "tokenize_tc_run: null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int dev = 0, sm_count = 0;
  RQB_CUDA(cudaGetDevice(&dev));
  RQB_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));     // per call: the state may live on any device
  // x's rows are bulk-copied to shared memory (16-byte aligned source and size): 16-byte aligned base and row pitch
  // (ops.py copies other layouts)
  RQB_CHECK_ARG(((ldx & 3) == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0),
                "tokenize_tc_run: x must be 16-byte aligned with a row stride that is a multiple of 4 floats");
  return tcx_run(x, ldx, B, state, D, K, L, ids, stats, sm_count, st);
}
