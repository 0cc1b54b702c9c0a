// Exact ranking of every corpus item for each history (modules/model.py EncoderDecoderRetrievalModel.rank_sem_ids / rank_items).
// Items that share an l-prefix share the causal decoder's state at positions 0..l, so one decoder row per node of the corpus
// trie (ops.SidPrefixIndex, per history) scores every corpus tuple.  The GEMMs are the split-precision tensor-core GEMM of
// csrc/gemm_tc.cu and the decoder step kernels of csrc/t5dec.cu (add-norm, self-attention through an ancestor table) are reused;
// these kernels do the rest:
//
//   rqb200_t5rank_cross_attention[_tc]  T5 cross-attention of Q queries per history (a trie level: up to tens of thousands) over
//                                  that history's encoder rows, t5rank_cross_attention_kernel<TF32>: one warpgroup per (64-query
//                                  tile, head, history), keys streamed through shared memory with an online fp32 softmax.  TF32:
//                                  64-key tiles, S = Q K^T by wgmma m64n64k8 from shared memory, O += P V with P as the register A
//                                  operand (the staging of csrc/t5_tc.cuh: a transposing V copy in the 0,2,4,6,1,3,5,7 key order).
//                                  fp32: the same query tiles on the CUDA cores, 32 keys per tile, the reference of the TF32 one.
//   rqb200_t5rank_children         after the level's head GEMM: one warp per node row computes the log-sum-exp exactly as
//                                  sid_beam_topk_kernel does (same formula, same reduction order), then writes every child's
//                                  score = parent score + (x[code] - lse).  A row with a NaN or +inf logit, or all -inf, is
//                                  counted and gives its children NaN.
//   rqb200_t5rank_select           one CTA per history over its U leaf scores: block radix selection of the n best leaves keyed
//                                  on (score descending, leaf ascending, NaN last), expansion of the chosen leaves to their items
//                                  in dedup order cut off at n, and the target item's rank as a block count.  No global atomics.
//
// Numerics are HF's T5 in eval mode: no 1/sqrt(d) scaling, an additive per-key mask (-FLT_MAX masks a key, as HF's eager mask).
#include <cfloat>

#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "sid_excl.cuh"
#include "t5_tc.cuh"

#define RK_DKV 64
#define RK_QTILE 64         // queries per CTA
#define RK_KTILE 32         // keys per shared-memory tile
#define RK_WARPS 4
#define RK_QPW (RK_QTILE / RK_WARPS)

__device__ __forceinline__ float rk_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------------ cross-attention
// grid (ceil(Q / 64), heads, B).  Query i of history b is row b * Q + i of q (head n at column n * 64); history b's keys are rows
// offsets[b] .. offsets[b + 1] - 1 of k / v, with additive key_mask[row] (null: 0).  Warp w owns queries w, w + 4, ... of the tile;
// in a key tile lane j scores key j, then lane d accumulates output dims d and d + 32.
template <bool TF32>
__global__ void __launch_bounds__(RK_WARPS * 32) t5rank_cross_attention_kernel(
    const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, const float* __restrict__ v, int64_t ldkv,
    const int* __restrict__ offsets, const float* __restrict__ key_mask, int Q, float* __restrict__ out, int64_t ldo);

// One fp32 query tile, head n = blockIdx.y, over history b's keys: queries qrow0 .. qrow0 + nq - 1 of q / out (nq <= 64).  The
// uniform kernel (RAGGED false: tile blockIdx.x of history blockIdx.z) and the ragged one (t5rank_cross_attention_ragged_kernel:
// tile blockIdx.x of the tile table) differ only in how a CTA finds (b, qrow0, nq), so a query's arithmetic does not depend on
// the layout.
template <bool RAGGED>
__device__ __forceinline__ void rk_cross_attention_tile(const float* __restrict__ q, int64_t ldq, const float* __restrict__ k,
                                                        const float* __restrict__ v, int64_t ldkv, const int* __restrict__ offsets,
                                                        const float* __restrict__ key_mask, int Q, const int* __restrict__ tiles,
                                                        float* __restrict__ out, int64_t ldo) {
  __shared__ float sq[RK_QTILE][RK_DKV];
  __shared__ float sk[RK_KTILE][RK_DKV + 1];   // +1: lane j reads row j, column d -> distinct banks
  __shared__ float sv[RK_KTILE][RK_DKV];
  __shared__ float sbias[RK_KTILE];
  int n, b, nq;
  int64_t col, qrow0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (RAGGED) {
    const int* tile = tiles + 3 * (int64_t)blockIdx.x;
    n = blockIdx.y;
    b = tile[0];
    nq = tile[2];
    col = (int64_t)n * RK_DKV;
    qrow0 = tile[1];
  } else {
    const int q0 = blockIdx.x * RK_QTILE;
    n = blockIdx.y;
    b = blockIdx.z;
    nq = min(RK_QTILE, Q - q0);
    col = (int64_t)n * RK_DKV;
    qrow0 = (int64_t)b * Q + q0;
  }
  for (int i = threadIdx.x; i < RK_QTILE * RK_DKV; i += blockDim.x) {
    const int r = i / RK_DKV, d = i % RK_DKV;
    sq[r][d] = r < nq ? q[(qrow0 + r) * ldq + col + d] : 0.f;
  }
  const int r0 = offsets[b], S = offsets[b + 1] - r0;

  float m[RK_QPW], l[RK_QPW], acc0[RK_QPW], acc1[RK_QPW];
#pragma unroll
  for (int t = 0; t < RK_QPW; ++t) { m[t] = -INFINITY; l[t] = 0.f; acc0[t] = 0.f; acc1[t] = 0.f; }

  const float* kb = k + (int64_t)r0 * ldkv + col;
  const float* vb = v + (int64_t)r0 * ldkv + col;
  for (int s0 = 0; s0 < S; s0 += RK_KTILE) {
    __syncthreads();                                        // the previous tile is consumed (and sq is written)
    for (int i = threadIdx.x; i < RK_KTILE * RK_DKV; i += blockDim.x) {
      const int j = i / RK_DKV, d = i % RK_DKV, s = s0 + j;
      sk[j][d] = s < S ? kb[(int64_t)s * ldkv + d] : 0.f;
      sv[j][d] = s < S ? vb[(int64_t)s * ldkv + d] : 0.f;
    }
    if (threadIdx.x < RK_KTILE) {
      const int s = s0 + threadIdx.x;
      sbias[threadIdx.x] = s >= S ? -INFINITY : (key_mask ? key_mask[r0 + s] : 0.f);
    }
    __syncthreads();
#pragma unroll
    for (int t = 0; t < RK_QPW; ++t) {
      const int qi = warp + t * RK_WARPS;
      if (qi >= nq) continue;
      float dot = 0.f;
#pragma unroll 16
      for (int d = 0; d < RK_DKV; ++d) dot = fmaf(sq[qi][d], sk[lane][d], dot);
      const float bias = sbias[lane];
      const float sc = bias == -INFINITY ? -INFINITY : dot + bias;   // a key past S contributes exp(-inf) = 0
      const float m_new = fmaxf(m[t], rk_warp_max(sc));              // finite: every tile holds at least one key < S
      const float alpha = expf(m[t] - m_new);
      const float p = expf(sc - m_new);
      l[t] = l[t] * alpha + warp_sum(p);
      float a0 = acc0[t] * alpha, a1 = acc1[t] * alpha;
#pragma unroll 8
      for (int j = 0; j < RK_KTILE; ++j) {
        const float pj = __shfl_sync(0xffffffffu, p, j);
        a0 = fmaf(pj, sv[j][lane], a0);
        a1 = fmaf(pj, sv[j][lane + 32], a1);
      }
      acc0[t] = a0;
      acc1[t] = a1;
      m[t] = m_new;
    }
  }
#pragma unroll
  for (int t = 0; t < RK_QPW; ++t) {
    const int qi = warp + t * RK_WARPS;
    if (qi >= nq) continue;
    float* o = out + (qrow0 + qi) * ldo + col;
    o[lane] = l[t] > 0.f ? acc0[t] / l[t] : 0.f;            // a history without keys gets zeros
    o[lane + 32] = l[t] > 0.f ? acc1[t] / l[t] : 0.f;
  }
}

template <>
__global__ void __launch_bounds__(RK_WARPS * 32) t5rank_cross_attention_kernel<false>(
    const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, const float* __restrict__ v, int64_t ldkv,
    const int* __restrict__ offsets, const float* __restrict__ key_mask, int Q, float* __restrict__ out, int64_t ldo) {
  rk_cross_attention_tile<false>(q, ldq, k, v, ldkv, offsets, key_mask, Q, nullptr, out, ldo);
}

// grid (T, heads): a ragged level, history b's queries the rows roff[b] .. roff[b + 1] - 1 of q.  Tile t is tiles[3 t ..] =
// (history, first query row, query count <= 64), as t5exact_frontier_kernel writes them.  LIVE: the grid is sized for T tiles (the
// capacity) and the tiles are the first *live; the CTAs of the others exit.
template <bool LIVE>
__global__ void __launch_bounds__(RK_WARPS * 32) t5rank_cross_attention_ragged_kernel(
    const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, const float* __restrict__ v, int64_t ldkv,
    const int* __restrict__ offsets, const float* __restrict__ key_mask, const int* __restrict__ tiles, float* __restrict__ out,
    int64_t ldo, const int* __restrict__ live) {
  if (LIVE && (int)blockIdx.x >= *live) return;
  rk_cross_attention_tile<true>(q, ldq, k, v, ldkv, offsets, key_mask, 0, tiles, out, ldo);
}


// The TF32 instantiation: the same grid and query tile, dynamic smem 3 tiles (Q, K, transposed V).  Thread (warp w, lane
// 4 g + t) holds query rows 16 w + g and 16 w + g + 8 of the tile and, of each 8-key block j, key columns 8 j + 2 t, 8 j + 2 t + 1.
// q, k, v rows must be 16-byte aligned with row strides a multiple of 4 floats.
extern __shared__ __align__(128) float rk_tc_smem[];

template <>
__global__ void __launch_bounds__(TC_THREADS) t5rank_cross_attention_kernel<true>(
    const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, const float* __restrict__ v, int64_t ldkv,
    const int* __restrict__ offsets, const float* __restrict__ key_mask, int Q, float* __restrict__ out, int64_t ldo) {
  float* sQ = rk_tc_smem;
  float* sK = sQ + TC_TILE;
  float* sVt = sK + TC_TILE;
  __shared__ float sbias[TC_T];
  const int q0 = blockIdx.x * TC_T, n = blockIdx.y, b = blockIdx.z;
  const int nq = min(TC_T, Q - q0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int row[2] = {16 * warp + g, 16 * warp + g + 8};
  const int64_t qrow0 = (int64_t)b * Q + q0;
  const int r0 = offsets[b], S = offsets[b + 1] - r0;
  tc_stage(sQ, q + qrow0 * ldq + n * 64, ldq, nq);
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  for (int t0 = 0; t0 < S; t0 += TC_T) {
    const int nk = min(TC_T, S - t0);
    __syncthreads();                                          // the previous tile's MMAs have completed in every warp
    tc_stage(sK, k + (int64_t)(r0 + t0) * ldkv + n * 64, ldkv, nk);
    tc_stage_t(sVt, v + (int64_t)(r0 + t0) * ldkv + n * 64, ldkv, nk);
    if (threadIdx.x < TC_T)
      sbias[threadIdx.x] = (int)threadIdx.x < nk ? (key_mask ? key_mask[r0 + t0 + threadIdx.x] : 0.f) : -INFINITY;
    tc_proxy_fence();
    __syncthreads();
    float s[32];
    tc_fence();
    tc_gemm_ss(s, sQ, sK);
    tc_commit();
    tc_wait();
    tc_pin(s);
    float mt[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float bias = sbias[8 * j + 2 * t + e];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float& x = s[4 * j + 2 * h + e];
          x = bias == -INFINITY ? -INFINITY : x + bias;       // a key past the history contributes exp(-inf) = 0
          mt[h] = fmaxf(mt[h], x);
        }
      }
    float alpha[2], lt[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mt[h] = fmaxf(mt[h], __shfl_xor_sync(0xffffffffu, mt[h], 1));
      mt[h] = fmaxf(mt[h], __shfl_xor_sync(0xffffffffu, mt[h], 2));
      const float m_new = fmaxf(m[h], mt[h]);                 // finite: every tile holds at least one key of the history
      alpha[h] = expf(m[h] - m_new);
      m[h] = m_new;
    }
    uint32_t a[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float p = expf(s[i] - m[(i >> 1) & 1]);
      lt[(i >> 1) & 1] += p;
      a[i] = tf32_bits(p);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l[h] = fmaf(l[h], alpha[h], lt[h]);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[4 * j] *= alpha[0];
      o[4 * j + 1] *= alpha[0];
      o[4 * j + 2] *= alpha[1];
      o[4 * j + 3] *= alpha[1];
    }
    tc_fence();
    tc_gemm_rs(o, a, sVt);
    tc_commit();
    tc_wait();
    tc_pin(o);
    tc_pin(a);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (row[h] >= nq) continue;
    float* orow = out + (qrow0 + row[h]) * ldo + n * 64 + 2 * t;
    const float inv_ok = l[h] > 0.f ? 1.f : 0.f;              // a history without keys gets zeros
    const float den = l[h] > 0.f ? l[h] : 1.f;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(o[4 * j + 2 * h] / den * inv_ok, o[4 * j + 2 * h + 1] / den * inv_ok);
  }
}

// cudaFuncSetAttribute once per device and kernel (bit d of *done: device d)
static int rk_set_smem_once(const void* fn, int bytes, unsigned long long* done) {
  int dev = 0;
  RQB_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && (*done >> dev) & 1ull) return RQB_OK;
  RQB_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  if (dev < 64) *done |= 1ull << dev;
  return RQB_OK;
}

static int rk_cross_attention(bool tf32, const char* what, const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv,
                              const int* offsets, const float* key_mask, int B, int Q, int heads, float* out, int64_t ldo,
                              void* stream) {
  RQB_CHECK_ARG(B >= 0 && Q >= 0 && heads > 0 && ldq >= (int64_t)heads * RK_DKV && ldkv >= (int64_t)heads * RK_DKV &&
                    ldo >= (int64_t)heads * RK_DKV,
                "%s: bad argument (B = %d, Q = %d, heads = %d)", what, B, Q, heads);
  if (B > 65535 || heads > 65535) {
    rqb_set_error("%s: need B <= 65535 and heads <= 65535 (B = %d, heads = %d)", what, B, heads);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0 || Q == 0) return RQB_OK;
  RQB_CHECK_ARG(q && k && v && offsets && out, "%s: null pointer", what);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid((unsigned)((Q + RK_QTILE - 1) / RK_QTILE), (unsigned)heads, (unsigned)B);
  if (tf32) {
    RQB_CHECK_ARG(ldq % 4 == 0 && ldkv % 4 == 0 && ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) |
                                                      reinterpret_cast<uintptr_t>(v)) & 15) == 0,
                  "%s: q, k, v must be 16-byte aligned with row strides a multiple of 4", what);
    static unsigned long long done = 0;
    const int smem = 3 * TC_TILE * (int)sizeof(float);
    const int rc = rk_set_smem_once(reinterpret_cast<const void*>(t5rank_cross_attention_kernel<true>), smem, &done);
    if (rc != RQB_OK) return rc;
    t5rank_cross_attention_kernel<true><<<grid, TC_THREADS, smem, st>>>(q, ldq, k, v, ldkv, offsets, key_mask, Q, out, ldo);
  } else {
    t5rank_cross_attention_kernel<false><<<grid, RK_WARPS * 32, 0, st>>>(q, ldq, k, v, ldkv, offsets, key_mask, Q, out, ldo);
  }
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5rank_cross_attention(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv,
                                             const int* offsets, const float* key_mask, int B, int Q, int heads, float* out,
                                             int64_t ldo, void* stream) {
  return rk_cross_attention(false, "t5rank_cross_attention", q, ldq, k, v, ldkv, offsets, key_mask, B, Q, heads, out, ldo, stream);
}

extern "C" int rqb200_t5rank_cross_attention_tc(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv,
                                                const int* offsets, const float* key_mask, int B, int Q, int heads, float* out,
                                                int64_t ldo, void* stream) {
  return rk_cross_attention(true, "t5rank_cross_attention_tc", q, ldq, k, v, ldkv, offsets, key_mask, B, Q, heads, out, ldo,
                            stream);
}

template <bool LIVE>
static int rk_ragged(const char* what, const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv, const int* offsets,
                     const float* key_mask, const int* tiles, int T, const int* live, int heads, float* out, int64_t ldo, void* stream) {
  RQB_CHECK_ARG(T >= 0 && heads > 0 && ldq >= (int64_t)heads * RK_DKV && ldkv >= (int64_t)heads * RK_DKV &&
                    ldo >= (int64_t)heads * RK_DKV,
                "%s: bad argument (T = %d, heads = %d)", what, T, heads);
  if (heads > 65535) {
    rqb_set_error("%s: need heads <= 65535 (heads = %d)", what, heads);
    return RQB_ERR_UNSUPPORTED;
  }
  if (T == 0) return RQB_OK;
  RQB_CHECK_ARG(q && k && v && offsets && tiles && out && (live || !LIVE), "%s: null pointer", what);
  t5rank_cross_attention_ragged_kernel<LIVE><<<dim3((unsigned)T, (unsigned)heads), RK_WARPS * 32, 0,
                                               reinterpret_cast<cudaStream_t>(stream)>>>(q, ldq, k, v, ldkv, offsets, key_mask, tiles,
                                                                                         out, ldo, live);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5rank_cross_attention_ragged(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv,
                                                    const int* offsets, const float* key_mask, const int* tiles, int T, int heads,
                                                    float* out, int64_t ldo, void* stream) {
  return rk_ragged<false>("t5rank_cross_attention_ragged", q, ldq, k, v, ldkv, offsets, key_mask, tiles, T, nullptr, heads, out, ldo,
                          stream);
}

extern "C" int rqb200_t5rank_cross_attention_ragged_counted(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv,
                                                            const int* offsets, const float* key_mask, const int* tiles, int T,
                                                            const int* live_t, int heads, float* out, int64_t ldo, void* stream) {
  return rk_ragged<true>("t5rank_cross_attention_ragged_counted", q, ldq, k, v, ldkv, offsets, key_mask, tiles, T, live_t, heads, out,
                         ldo, stream);
}

// ------------------------------------------------------------------------------------------------ children scores
// One warp per node row r = b * n_h + i of logits [R, K].  lse as sid_beam_topk_kernel: m = max, sum of expf(x - m) over c = lane,
// lane + 32, ... then an xor butterfly (every lane ends with the same bits), lse = m + logf(sum).  Child j of node i (child[i] <=
// j < child[i + 1], a node of level h + 1) gets out[b * n_next + j] = (x[code[j]] - lse) + parent[r] with explicit roundings.
// LIVE: one group (n_h = R) whose rows are the first min(live[0], R) of the grid's R (the capacity); the warps of the others
// exit.  live[1], the group's children, is what child[] ranges over: with one group it offsets nothing.
template <bool LIVE>
__global__ void __launch_bounds__(256) t5rank_children_kernel(const float* __restrict__ logits, int64_t ld, int R, int K, int n_h,
                                                              const float* __restrict__ parent, const int* __restrict__ child,
                                                              const int* __restrict__ code, int n_next, float* __restrict__ out,
                                                              int* __restrict__ bad, const int* __restrict__ live) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (LIVE) R = min(R, max(0, live[0]));
  if (r >= R) return;
  const int64_t b = r / n_h;
  const int i = (int)(r - b * n_h);
  const float* x = logits + r * ld;
  float m = -INFINITY;
  bool odd = false;
  for (int c = lane; c < K; c += 32) {
    const float val = x[c];
    m = fmaxf(m, val);
    odd |= val != val || val == INFINITY;
  }
  m = rk_warp_max(m);
  odd = __any_sync(0xffffffffu, odd);
  float sum = 0.f;
  for (int c = lane; c < K; c += 32) sum += expf(x[c] - m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float lse = m + logf(sum);
  const bool nonfinite = odd || m == -INFINITY;
  if (nonfinite && lane == 0 && bad) atomicAdd(bad, 1);
  const float ps = parent ? parent[r] : 0.f;
  float* o = out + b * n_next;
  for (int j = child[i] + lane; j < child[i + 1]; j += 32)
    o[j] = nonfinite ? __int_as_float(0x7fffffff) : __fadd_rn(__fsub_rn(x[code[j]], lse), ps);
}

extern "C" int rqb200_t5rank_children(const float* logits, int64_t ld, int R, int K, int n_h, const float* parent, const int* child,
                                      const int* code, int n_next, float* out, int* bad, void* stream) {
  RQB_CHECK_ARG(R >= 0 && K > 0 && n_h > 0 && n_next >= 0 && ld >= K && R % n_h == 0,
                "t5rank_children: bad argument (R = %d, K = %d, n_h = %d, n_next = %d)", R, K, n_h, n_next);
  if (R == 0) return RQB_OK;
  RQB_CHECK_ARG(logits && child && code && out, "t5rank_children: null pointer");
  const int rows_per_block = 8;
  t5rank_children_kernel<false><<<(R + rows_per_block - 1) / rows_per_block, rows_per_block * 32, 0,
                                  reinterpret_cast<cudaStream_t>(stream)>>>(logits, ld, R, K, n_h, parent, child, code, n_next, out,
                                                                            bad, nullptr);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5rank_children_counted(const float* logits, int64_t ld, int R, int K, const float* parent, const int* child,
                                              const int* code, int n_next, const int* live, float* out, int* bad, void* stream) {
  RQB_CHECK_ARG(R >= 0 && K > 0 && n_next >= 0 && ld >= K, "t5rank_children_counted: bad argument (R = %d, K = %d, n_next = %d)", R,
                K, n_next);
  if (R == 0) return RQB_OK;
  RQB_CHECK_ARG(logits && child && code && out && live, "t5rank_children_counted: null pointer");
  const int rows_per_block = 8;
  t5rank_children_kernel<true><<<(R + rows_per_block - 1) / rows_per_block, rows_per_block * 32, 0,
                                 reinterpret_cast<cudaStream_t>(stream)>>>(logits, ld, R, K, R, parent, child, code, n_next, out, bad,
                                                                           live);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ------------------------------------------------------------------------------------------------ per-history selection
// Order key of a leaf: its score's order-preserving 32-bit image (-0 folded into +0, NaN mapped to 0, below every number) above
// 0xffffffff - leaf, so keys are distinct and "descending key" is (score descending, leaf ascending, NaN last).
#define RK_SEL_THREADS 512
#define RK_SEL_MAX_N 1024
#define RK_SEL_SMEM_KEYS (24 * 1024)

__device__ __forceinline__ unsigned int rk_score_key(float v) {
  if (v != v) return 0u;
  const unsigned int x = __float_as_uint(v == 0.f ? 0.f : v);
  return x ^ ((x & 0x80000000u) ? 0xffffffffu : 0x80000000u);
}

__device__ __forceinline__ unsigned long long rk_key64(unsigned int key, int leaf) {
  return ((unsigned long long)key << 32) | (unsigned int)(0xffffffffu - (unsigned int)leaf);
}

// With an exclusion (EXCL): a leaf whose items are all excluded takes the key RK_BLOCKED, which rk_score_key never returns, and
// no part in the selection.  Thread-strided passes meet leaves in ascending order, so a thread finds whether its leaf is blocked
// with a cursor over the excluded positions' leaves (ascending): O(U / threads + excluded) per pass.
#define RK_BLOCKED 1u

struct RkBlockedCursor {
  int c = 0;
  __device__ __forceinline__ bool at(int u, const int* x_leaf, const unsigned char* x_full, int nx) {
    while (c < nx && x_leaf[c] < u) ++c;
    return c < nx && x_leaf[c] == u && x_full[c];
  }
};

// Radix selection of the nsel-th largest 32-bit key among entries u = 0 .. U - 1 (key_of(u); with SKIP, entries whose key is
// RK_BLOCKED take no part): 8-bit digits from the top, stopping once the chosen bin is taken whole.  Leaves in prefix / pmask
// the chosen key bits and in want how many entries at that prefix are taken (the caller takes the lowest-index ones).  Each pass
// meets u in ascending order per thread, after key_of.restart().  hist [256] is zero on entry and on return; ctl holds 3 ints.
template <bool SKIP, typename KeyOf>
__device__ __forceinline__ void rk_radix_threshold(int U, int nsel, KeyOf& key_of, int* hist, int* ctl, unsigned int& prefix,
                                                   unsigned int& pmask, int& want) {
  const int nt = RK_SEL_THREADS, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned int lt = (1u << lane) - 1u;
  prefix = 0;
  pmask = 0;
  want = nsel;
  for (int shift = 24; shift >= 0 && nsel > 0; shift -= 8) {
    key_of.restart();
    for (int base = 0; base < U; base += nt) {
      const int u = base + threadIdx.x;
      int d = 256;
      if (u < U) {
        const unsigned int key = key_of(u);
        if ((key & pmask) == prefix && !(SKIP && key == RK_BLOCKED)) d = (int)((key >> shift) & 255u);
      }
      const unsigned int same = __match_any_sync(0xffffffffu, d);
      if (d < 256 && (same & lt) == 0) atomicAdd(&hist[d], __popc(same));   // integer counts: order does not matter
    }
    __syncthreads();
    if (w == 0) {
      int c[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = hist[lane * 8 + j];
        hist[lane * 8 + j] = 0;
        sum += c[j];
      }
      int suf = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_down_sync(0xffffffffu, suf, o);
        if (lane + o < 32) suf += t;
      }
      const int owner = 31 - __clz(__ballot_sync(0xffffffffu, suf >= want));
      if (lane == owner) {
        int acc = suf - sum;
        for (int j = 7; j >= 0; --j) {
          if (acc + c[j] >= want) {
            ctl[0] = lane * 8 + j;
            ctl[1] = acc;
            ctl[2] = c[j];
            break;
          }
          acc += c[j];
        }
      }
    }
    __syncthreads();
    want -= ctl[1];
    prefix |= (unsigned int)ctl[0] << shift;
    pmask |= 255u << shift;
    const bool whole = ctl[2] == want;
    __syncthreads();                                        // ctl is read by every thread before the next pass writes it
    if (whole) break;
  }
}

// t5rank_select_kernel's leaf keys: from shared memory, or from the scores with the blocked-leaf cursor
template <bool KEYS_IN_SMEM, bool EXCL>
struct RkLeafKeys {
  const unsigned int* s_key;
  const float* sc;
  const int* x_leaf;
  const unsigned char* x_full;
  int nx;
  RkBlockedCursor cur;
  __device__ __forceinline__ void restart() { cur = RkBlockedCursor(); }
  __device__ __forceinline__ unsigned int operator()(int u) {
    return KEYS_IN_SMEM ? s_key[u] : (EXCL && cur.at(u, x_leaf, x_full, nx)) ? RK_BLOCKED : rk_score_key(sc[u]);
  }
};

template <bool KEYS_IN_SMEM, bool EXCL>
__global__ void __launch_bounds__(RK_SEL_THREADS) t5rank_select_kernel(
    const float* __restrict__ scores, int U, const int* __restrict__ row, const int* __restrict__ start,
    const int64_t* __restrict__ t_leaf, const int64_t* __restrict__ t_dedup, int n, int64_t* __restrict__ out_items,
    float* __restrict__ out_scores, int64_t* __restrict__ out_rank, SidExcl ex) {
  using Scan = cub::BlockScan<int, RK_SEL_THREADS>;
  using Reduce = cub::BlockReduce<long long, RK_SEL_THREADS>;
  __shared__ union {
    typename Scan::TempStorage scan;
    typename Reduce::TempStorage reduce;
  } tmp;
  __shared__ int hist[256];
  __shared__ int ctl[3];                                    // chosen digit, entries above its bin, entries in its bin
  __shared__ int nsel_at, ties_base;
  __shared__ unsigned long long sel[RK_SEL_MAX_N];
  __shared__ int s_leaf[RK_SEL_MAX_N];
  __shared__ int s_off[RK_SEL_MAX_N + 1];
  __shared__ int x_leaf[EXCL ? SID_EXCL_MAX_M : 1];         // the leaf of each excluded position
  __shared__ unsigned char x_full[EXCL ? SID_EXCL_MAX_M : 1];   // ... and whether that leaf's items are all excluded
  __shared__ int n_blocked;
  extern __shared__ __align__(16) unsigned int s_key[];     // [U] when KEYS_IN_SMEM
  const int nt = RK_SEL_THREADS;
  const int64_t b = blockIdx.x;
  const float* sc = scores + b * U;
  const int* xp = EXCL ? ex.pos_of(b) : nullptr;            // the history's excluded positions, ascending
  const int nx = EXCL ? ex.npos(b) : 0;
  for (int i = threadIdx.x; i < 256; i += nt) hist[i] = 0;
  if (threadIdx.x == 0) {
    nsel_at = 0;
    ties_base = 0;
    n_blocked = 0;
  }
  if (EXCL) {
    __syncthreads();
    for (int i = threadIdx.x; i < nx; i += nt) {
      const int r = xp[i];
      int lo = 0, hi = U;                                   // the leaf u with start[u] <= r < start[u + 1]
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (start[mid] <= r) lo = mid;
        else hi = mid;
      }
      const int s = start[lo], e = start[lo + 1];
      const bool full = sid_excluded_in(xp, nx, s, e) == e - s;
      x_leaf[i] = lo;
      x_full[i] = full ? 1 : 0;
      if (full && (i == 0 || xp[i - 1] < s)) atomicAdd(&n_blocked, 1);   // an integer count: order does not matter
    }
    __syncthreads();
  }
  const int nsel = min(n, U - (EXCL ? n_blocked : 0));
  if (KEYS_IN_SMEM) {
    RkBlockedCursor cur;
    for (int u = threadIdx.x; u < U; u += nt)
      s_key[u] = (EXCL && cur.at(u, x_leaf, x_full, nx)) ? RK_BLOCKED : rk_score_key(sc[u]);
  }
  __syncthreads();
  unsigned int prefix, pmask;
  int want;
  RkLeafKeys<KEYS_IN_SMEM, EXCL> key_of{s_key, sc, x_leaf, x_full, nx};
  rk_radix_threshold<EXCL>(U, nsel, key_of, hist, ctl, prefix, pmask, want);
  // keep every leaf above the threshold and the `want` lowest-index leaves at it (an ordered block scan over the ties), and count
  // the items of the leaves that sort before the target
  const int64_t tl = t_leaf[b];
  int64_t td = t_dedup[b];
  bool t_ok = tl >= 0 && tl < U && td >= 0 && td < (int64_t)(start[tl + 1] - start[tl]);
  if (EXCL && t_ok) {                                       // the target's position among its leaf's items that are not excluded
    const int r = start[tl] + (int)td;
    const int at = sid_lower_bound(xp, nx, r);
    t_ok = !(at < nx && xp[at] == r);
    td -= at - sid_lower_bound(xp, nx, start[tl]);
  }
  const unsigned long long t_key = t_ok ? rk_key64(KEYS_IN_SMEM ? s_key[tl] : rk_score_key(sc[tl]), (int)tl) : 0ull;
  long long before = 0;
  if (EXCL && t_ok)                                         // the excluded items of the leaves counted below
    for (int i = threadIdx.x; i < nx; i += nt) {
      const int u = x_leaf[i];
      const unsigned int key = KEYS_IN_SMEM ? s_key[u] : x_full[i] ? RK_BLOCKED : rk_score_key(sc[u]);
      if (rk_key64(key, u) > t_key) --before;
    }
  RkBlockedCursor cur;
  for (int base = 0; base < U; base += nt) {
    const int u = base + threadIdx.x;
    unsigned int key = 0;
    if (u < U) key = KEYS_IN_SMEM ? s_key[u] : (EXCL && cur.at(u, x_leaf, x_full, nx)) ? RK_BLOCKED : rk_score_key(sc[u]);
    const bool in = u < U && nsel > 0 && !(EXCL && key == RK_BLOCKED);
    const bool above = in && (key & pmask) > prefix;
    const int tie = (in && (key & pmask) == prefix) ? 1 : 0;
    int excl, total;
    Scan(tmp.scan).ExclusiveSum(tie, excl, total);
    const bool take = above || (tie && ties_base + excl < want);
    if (take) {
      const int at = atomicAdd(&nsel_at, 1);                // a slot only: the final order is each key's rank below
      sel[at] = rk_key64(key, u);
    }
    if (t_ok && u < U && rk_key64(key, u) > t_key) before += start[u + 1] - start[u];
    __syncthreads();                                        // scan storage and ties_base reused
    if (threadIdx.x == 0) ties_base += total;
    __syncthreads();
  }
  const long long items_before = Reduce(tmp.reduce).Sum(before);
  __syncthreads();
  // rank each kept key among the kept ones (distinct keys), then each leaf's item count, scanned in rank order
  for (int i = threadIdx.x; i < nsel; i += nt) {
    const unsigned long long key = sel[i];
    int r = 0;
    for (int j = 0; j < nsel; ++j) r += sel[j] > key;
    s_leaf[r] = (int)(0xffffffffu - (unsigned int)(key & 0xffffffffull));
  }
  __syncthreads();
  constexpr int PER = RK_SEL_MAX_N / RK_SEL_THREADS;
  int cnt[PER], off[PER], total;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int j = threadIdx.x * PER + i;
    cnt[i] = 0;
    if (j < nsel) {
      const int s = start[s_leaf[j]], e = start[s_leaf[j] + 1];
      cnt[i] = e - s - (EXCL ? sid_excluded_in(xp, nx, s, e) : 0);
    }
  }
  Scan(tmp.scan).ExclusiveSum(cnt, off, total);
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int j = threadIdx.x * PER + i;
    if (j < nsel) s_off[j] = off[i];
  }
  __syncthreads();
  const int mcount = min(total, n);
  for (int o = threadIdx.x; o < n; o += nt) {
    int64_t item = -1;
    float s = -INFINITY;
    if (o < mcount) {                                       // s_off[lo] <= o < s_off[lo + 1]: leaf lo holds slot o
      int lo = 0, hi = nsel;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_off[mid] <= o) lo = mid;
        else hi = mid;
      }
      const int leaf = s_leaf[lo];
      item = row[EXCL ? sid_nth_kept(xp, nx, start[leaf], o - s_off[lo]) : start[leaf] + (o - s_off[lo])];
      s = sc[leaf];
    }
    out_items[b * n + o] = item;
    out_scores[b * n + o] = s;
  }
  if (threadIdx.x == 0) out_rank[b] = t_ok ? (int64_t)items_before + td : -1;
}

template <bool EXCL>
static int rk_select(const float* scores, int B, int U, const int* row, const int* start, const int64_t* t_leaf, const int64_t* t_dedup,
                     int n, int64_t* out_items, float* out_scores, int64_t* out_rank, const SidExcl& ex, void* stream) {
  RQB_CHECK_ARG(B >= 0 && U >= 0 && n > 0, "t5rank_select: bad argument (B = %d, U = %d, n = %d)", B, U, n);
  if (n > RK_SEL_MAX_N) {
    rqb_set_error("t5rank_select: need n <= %d (n = %d)", RK_SEL_MAX_N, n);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG((scores || U == 0) && start && (row || U == 0) && t_leaf && t_dedup && out_items && out_scores && out_rank,
                "t5rank_select: null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (U <= RK_SEL_SMEM_KEYS) {
    const size_t smem = (size_t)U * sizeof(unsigned int);
    static unsigned long long done = 0;
    const int rc = rk_set_smem_once(reinterpret_cast<const void*>(t5rank_select_kernel<true, EXCL>),
                                    RK_SEL_SMEM_KEYS * (int)sizeof(unsigned int), &done);
    if (rc != RQB_OK) return rc;
    t5rank_select_kernel<true, EXCL><<<B, RK_SEL_THREADS, smem, st>>>(scores, U, row, start, t_leaf, t_dedup, n, out_items,
                                                                     out_scores, out_rank, ex);
  } else {
    t5rank_select_kernel<false, EXCL><<<B, RK_SEL_THREADS, 0, st>>>(scores, U, row, start, t_leaf, t_dedup, n, out_items,
                                                                   out_scores, out_rank, ex);
  }
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5rank_select(const float* scores, int B, int U, const int* row, const int* start, const int64_t* t_leaf,
                                    const int64_t* t_dedup, int n, int64_t* out_items, float* out_scores, int64_t* out_rank,
                                    void* stream) {
  return rk_select<false>(scores, B, U, row, start, t_leaf, t_dedup, n, out_items, out_scores, out_rank, SidExcl{}, stream);
}

extern "C" int rqb200_t5rank_select_excluding(const float* scores, int B, int U, const int* row, const int* start,
                                              const int64_t* t_leaf, const int64_t* t_dedup, int n, int64_t* out_items,
                                              float* out_scores, int64_t* out_rank, const int* ex_pos, const int64_t* ex_blocked,
                                              const int* ex_count, int ex_M, int ex_H, void* stream) {
  RQB_CHECK_ARG(ex_pos && ex_count && ex_M > 0 && ex_M <= SID_EXCL_MAX_M && ex_H > 0 && ex_H <= RQB_MAX_LEVELS,
                "t5rank_select_excluding: bad exclusion (M = %d, H = %d, need M <= %d)", ex_M, ex_H, SID_EXCL_MAX_M);
  const SidExcl ex{ex_pos, reinterpret_cast<const long long*>(ex_blocked), ex_count, ex_M, ex_H};
  return rk_select<true>(scores, B, U, row, start, t_leaf, t_dedup, n, out_items, out_scores, out_rank, ex, stream);
}

// ------------------------------------------------------------------------------------------------ per-history candidate trie
// Exact scoring of given tuples (modules/model.py score_sem_ids / score_items) decodes, per history, the trie of that history's
// C candidates instead of the corpus's.  One CTA per history: each candidate packs into a 64-bit key (bits = bits(K - 1) per id,
// the first id highest, so key order is lexicographic); a tuple with an id outside [0, K) gets the key 1 << (H bits), above every
// valid key.  A block radix sort (stable: equal keys stay in candidate order) over bits 0 .. H bits, then per level l = 1..H the
// distinct l-prefixes are flagged and numbered by a block scan.  Writes are plain stores to distinct addresses: no atomics, the
// output is a function of the input alone.
#define SC_THREADS 512
#define SC_MAX_C 4096

template <int IPT>
__global__ void __launch_bounds__(SC_THREADS) t5score_trie_kernel(const int64_t* __restrict__ ids, int C, int H, int K, int bits,
                                                                  int* __restrict__ counts, int* __restrict__ code,
                                                                  int* __restrict__ parent, int* __restrict__ child,
                                                                  int* __restrict__ leaf) {
  using Sort = cub::BlockRadixSort<unsigned long long, SC_THREADS, IPT, int>;
  using Scan = cub::BlockScan<int, SC_THREADS>;
  __shared__ union {
    typename Sort::TempStorage sort;
    typename Scan::TempStorage scan;
  } tmp;
  __shared__ unsigned long long s_last[SC_THREADS];
  const int64_t b = blockIdx.x;
  const int tid = threadIdx.x;
  const int vbits = H * bits;
  const unsigned long long invalid = 1ull << vbits;
  const int64_t* in = ids + b * (int64_t)C * H;
  unsigned long long key[IPT];
  int idx[IPT];
#pragma unroll
  for (int j = 0; j < IPT; ++j) {                           // blocked: thread t holds candidates t IPT .. t IPT + IPT - 1
    const int c = tid * IPT + j;
    idx[j] = c;
    key[j] = invalid;
    if (c < C) {
      unsigned long long k = 0;
      bool ok = true;
      for (int h = 0; h < H; ++h) {
        const int64_t v = in[(int64_t)c * H + h];
        ok &= v >= 0 && v < K;
        k = (k << bits) | (unsigned long long)(ok ? v : 0);
      }
      if (ok) key[j] = k;
    }
  }
  Sort(tmp.sort).Sort(key, idx, 0, vbits + 1);
  __syncthreads();
  s_last[tid] = key[IPT - 1];
  __syncthreads();
  const unsigned long long before = tid > 0 ? s_last[tid - 1] : invalid;
  int* cnt_out = counts + b * H;
  int prev_node[IPT], cnt_prev = 1;                         // level l - 1: every valid candidate's node; the root is node 0
  bool prev_flag[IPT];
#pragma unroll
  for (int j = 0; j < IPT; ++j) {
    prev_node[j] = 0;
    prev_flag[j] = false;
  }
  if (tid == 0) child[b * H * (C + 1)] = 0;                 // the root's children start at node 0 of level 1
  for (int l = 1; l <= H; ++l) {
    const int shift = (H - l) * bits;
    int flag[IPT], node[IPT], total;
#pragma unroll
    for (int j = 0; j < IPT; ++j) {
      const unsigned long long prev = j > 0 ? key[j - 1] : before;
      const bool valid = key[j] < invalid;
      flag[j] = valid && (prev >= invalid || (prev >> shift) != (key[j] >> shift)) ? 1 : 0;
    }
    Scan(tmp.scan).InclusiveSum(flag, node, total);
    __syncthreads();                                        // scan storage is reused by the next level
    int* lcode = code + (b * H + (l - 1)) * (int64_t)C;
    int* lpar = parent + (b * H + (l - 1)) * (int64_t)C;
    int* pchild = child + (b * H + (l - 1)) * (int64_t)(C + 1);   // level l - 1's child ranges
#pragma unroll
    for (int j = 0; j < IPT; ++j) {
      node[j] -= 1;
      if (flag[j]) {
        lcode[node[j]] = (int)((key[j] >> shift) & ((1ull << bits) - 1ull));
        lpar[node[j]] = prev_node[j];
        if (l > 1 && prev_flag[j]) pchild[prev_node[j]] = node[j];   // the first child of a new (l - 1)-prefix
      }
    }
    for (int i = total + tid; i < C; i += SC_THREADS) {     // padding nodes: a valid code and parent
      lcode[i] = 0;
      lpar[i] = 0;
    }
    for (int i = cnt_prev + tid; i <= C; i += SC_THREADS) pchild[i] = total;
    if (tid == 0) cnt_out[l - 1] = total;
#pragma unroll
    for (int j = 0; j < IPT; ++j) {
      prev_node[j] = node[j];
      prev_flag[j] = flag[j] != 0;
    }
    cnt_prev = total;
  }
  int* lf = leaf + b * C;
#pragma unroll
  for (int j = 0; j < IPT; ++j)
    if (idx[j] < C) lf[idx[j]] = key[j] < invalid ? prev_node[j] : -1;
}

extern "C" int rqb200_t5score_trie_build(const int64_t* ids, int B, int C, int H, int K, int* counts, int* code, int* parent,
                                         int* child, int* leaf, void* stream) {
  RQB_CHECK_ARG(B >= 0 && C > 0 && H > 0 && K > 0, "t5score_trie_build: bad argument (B = %d, C = %d, H = %d, K = %d)", B, C, H, K);
  int bits = 1;
  while (bits < 31 && (1 << bits) < K) ++bits;              // bits(K - 1), at least 1
  if (C > SC_MAX_C || H > RQB_MAX_LEVELS || H * bits > 62) {
    rqb_set_error("t5score_trie_build: need C <= %d, H <= %d and H * bits(K - 1) <= 62 (C = %d, H = %d, K = %d)", SC_MAX_C,
                  RQB_MAX_LEVELS, C, H, K);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(ids && counts && code && parent && child && leaf, "t5score_trie_build: null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (C <= SC_THREADS)
    t5score_trie_kernel<1><<<B, SC_THREADS, 0, st>>>(ids, C, H, K, bits, counts, code, parent, child, leaf);
  else if (C <= 2 * SC_THREADS)
    t5score_trie_kernel<2><<<B, SC_THREADS, 0, st>>>(ids, C, H, K, bits, counts, code, parent, child, leaf);
  else if (C <= 4 * SC_THREADS)
    t5score_trie_kernel<4><<<B, SC_THREADS, 0, st>>>(ids, C, H, K, bits, counts, code, parent, child, leaf);
  else
    t5score_trie_kernel<8><<<B, SC_THREADS, 0, st>>>(ids, C, H, K, bits, counts, code, parent, child, leaf);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ------------------------------------------------------------------------------------------------ exact top-k search
// The pruned exact decode of generate(search="exact") (modules/model.py FusedT5Exact).  A child never scores above its parent
// (t5rank_children adds a log-probability <= 0), so with tau[b] the score of some b-th history's w-th best valid leaf already
// known, a node scoring below tau[b] has no descendant in the exact top w.  Per level, after t5rank_children:
//
//   rqb200_t5exact_frontier[_excluding/_including]  one CTA per history over its scored children (nodes of trie level l): keeps
//                                  each child with score >= tau[b] that the history's filter does not block (the binary searches of
//                                  sid_excl.cuh in the level-l keys), block-scans the kept flags and the kept nodes' child counts,
//                                  and writes the next decoder level's rows (ragged: history b's are roff[b] .. roff[b + 1] - 1, in
//                                  trie order), their cross-attention query tiles, and the kept nodes' children (level l + 1) as one
//                                  group of compact child ranges, codes, node ids and parent rows for t5rank_children.  Two phases
//                                  from the same flags: a count pass (per history: kept rows, their children, query tiles), a scan
//                                  and a host read of the totals by the caller, then a write pass at the scanned offsets.
//   rqb200_t5exact_select[_excluding/_including]    one CTA per history over its leaf candidates (the children of the last
//                                  decoded level): rk_radix_threshold selection of the w best keys rk_key64(score, candidate) --
//                                  candidates are in leaf order, so (score descending, leaf ascending) -- with blocked and NaN leaves
//                                  left out, then each chosen leaf's tuple (read along its trie path) and score, -1 / -inf past the
//                                  valid candidates.
// Plain stores only, no global atomics: each output is a function of the input.
#define EX_THREADS 256

// whether history b's level-l list of the filter holds key (ascending keys)
__device__ __forceinline__ bool ex_listed(const SidExcl& f, int64_t b, int l, long long key) {
  const long long* list = f.keys_of(b, l);
  const int n = f.nkeys(b, l);
  const int i = sid_lower_bound(list, n, key);
  return i < n && __ldg(list + i) == key;
}

// whether the l-prefix key is invalid for history b under the consumer's filter mode
template <int FILTER>
__device__ __forceinline__ bool ex_blocked(const SidExcl& f, int64_t b, int l, long long key) {
  if (FILTER == SID_FILTER_EXCLUDE) return ex_listed(f, b, l, key);
  if (FILTER == SID_FILTER_INCLUDE) return !ex_listed(f, b, l, key);
  return false;
}

// Children of history b: entries coff[b] .. coff[b + 1] - 1 of sc / cnode / ccode / cpar, or with cnode null (the root's children,
// level 1) entries b n_root .. b n_root + n_root - 1 of sc, child i being node i of level 1 (code ccode[i], parent row b).
// pkey [rows]: the prefix key of each parent row (null at level 1).  counts (count pass) int32 [3, Bc]; offs (write pass) int32
// [3, Bc + 1], the exclusive scans of counts.
// CAP (the write pass of rqb200_t5exact_frontier_capacity*, for a caller that cannot read the totals on the host): the outputs
// hold cap.r rows, cap.c children and cap.t tiles.  Every CTA reads the totals offs[., Bc]; when they fit, the pass writes what
// the plain write pass writes, plus cap.live = the totals (R, C, T) and cap.noff [Bc + 1] = offs[1] (the children's offsets, which
// the next level's passes read).  When a total exceeds its capacity it writes no row, sets cap.live and cap.noff to 0 -- the next
// levels then see no rows -- and sets *cap.overflow = 1.
struct ExCap {
  int r, c, t;
  int* live;
  int* overflow;
  int* noff;
};

template <int FILTER, bool WRITE, bool CAP>
__global__ void __launch_bounds__(EX_THREADS) t5exact_frontier_kernel(
    const float* __restrict__ sc, const int* __restrict__ coff, int n_root, const int* __restrict__ cnode,
    const int* __restrict__ ccode, const int* __restrict__ cpar, const long long* __restrict__ pkey, const float* __restrict__ tau,
    int Bc, int K, int l, const int* __restrict__ lchild, const int* __restrict__ lcode_next, SidExcl f, int b0,
    int* __restrict__ counts, const int* __restrict__ offs, int64_t* __restrict__ row_code, int64_t* __restrict__ row_par,
    float* __restrict__ row_score, long long* __restrict__ row_key, int* __restrict__ row_node, int* __restrict__ tiles,
    int* __restrict__ nrng, int* __restrict__ nnode, int* __restrict__ ncode, int* __restrict__ npar, ExCap cap) {
  using Scan = cub::BlockScan<long long, EX_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ long long carry;                               // (kept rows << 32) + their children, of the tiles before
  const int b = blockIdx.x;
  const int64_t bg = (int64_t)b0 + b;
  const bool root = cnode == nullptr;
  const int64_t cs = root ? (int64_t)b * n_root : coff[b], ce = root ? cs + n_root : coff[b + 1];
  const float t = tau[b];
  int roff = 0, cbase = 0, toff = 0;
  if (WRITE) {
    roff = offs[b];
    cbase = offs[(Bc + 1) + b];
    toff = offs[2 * (Bc + 1) + b];
  }
  if (CAP) {
    const int R = offs[Bc], C = offs[2 * (Bc + 1) - 1], T = offs[3 * (Bc + 1) - 1];
    const bool over = R > cap.r || C > cap.c || T > cap.t;
    if (threadIdx.x == 0) {
      cap.noff[b] = over ? 0 : cbase;
      if (b == Bc - 1) cap.noff[Bc] = over ? 0 : C;
      if (b == 0) {
        cap.live[0] = over ? 0 : R;
        cap.live[1] = over ? 0 : C;
        cap.live[2] = over ? 0 : T;
        if (over) *cap.overflow = 1;
      }
    }
    if (over) return;
  }
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t base = cs; base < ce; base += EX_THREADS) {
    const int64_t j = base + threadIdx.x;
    long long flag = 0, key = 0;
    int node = 0, code = 0, par = 0;
    float s = 0.f;
    if (j < ce) {
      node = root ? (int)(j - cs) : cnode[j];
      code = root ? ccode[node] : ccode[j];
      par = root ? b : cpar[j];
      s = sc[j];
      bool keep = s >= t;                                   // NaN: never kept
      if (FILTER != SID_FILTER_NONE) {
        key = (root ? 0ll : pkey[par] * K) + code;
        keep = keep && !ex_blocked<FILTER>(f, bg, l, key);
      }
      if (keep) flag = (1ll << 32) + (lchild[node + 1] - lchild[node]);
    }
    long long excl, total;
    Scan(tmp).ExclusiveSum(flag, excl, total);
    const long long at = carry + excl;
    if (WRITE && flag) {
      const int row = roff + (int)(at >> 32);
      row_code[row] = code;
      row_par[row] = par;
      row_score[row] = s;
      if (FILTER != SID_FILTER_NONE) row_key[row] = key;
      row_node[row] = node;
      nrng[row] = cbase + (int)(at & 0xffffffffll);
    }
    __syncthreads();                                        // carry read and scan storage used by every thread
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
  const int kept = (int)(carry >> 32), nch = (int)(carry & 0xffffffffll);
  const int ntile = (kept + RK_QTILE - 1) / RK_QTILE;
  if constexpr (!WRITE) {
    if (threadIdx.x == 0) {
      counts[b] = kept;
      counts[Bc + b] = nch;
      counts[2 * Bc + b] = ntile;
    }
  } else {
    for (int i = threadIdx.x; i < ntile; i += EX_THREADS) {
      int* tile = tiles + 3 * (int64_t)(toff + i);
      tile[0] = b;
      tile[1] = roff + i * RK_QTILE;
      tile[2] = min(RK_QTILE, kept - i * RK_QTILE);
    }
    if (b == Bc - 1 && threadIdx.x == 0) nrng[roff + kept] = cbase + nch;   // the closing range entry
    __syncthreads();                                          // this history's nrng / row_node entries are written
    // child c of the history: in the range of the last kept row starting at or before it (ranges are ascending)
    for (int c = threadIdx.x; c < nch; c += EX_THREADS) {
      const int g = cbase + c;
      int lo = 0, hi = kept;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (nrng[roff + mid] <= g) lo = mid;
        else hi = mid;
      }
      const int row = roff + lo;
      const int child = lchild[row_node[row]] + (g - nrng[row]);
      nnode[g] = child;
      ncode[g] = lcode_next[child];
      npar[g] = row;
    }
  }
}

// t5exact_select_kernel's candidate keys: rk_score_key of the score, RK_BLOCKED for NaN and for leaves the filter blocks
template <bool KEYS_IN_SMEM, int FILTER>
struct ExLeafKeys {
  const unsigned int* s_key;
  const float* sc;
  const int* cnode;
  const long long* leaf_key;
  SidExcl f;
  int64_t b;
  int H;
  __device__ __forceinline__ void restart() {}
  __device__ __forceinline__ unsigned int compute(int u) const {
    const float s = sc[u];
    if (s != s) return RK_BLOCKED;
    if (FILTER != SID_FILTER_NONE && ex_blocked<FILTER>(f, b, H, leaf_key[cnode ? cnode[u] : u])) return RK_BLOCKED;
    return rk_score_key(s);
  }
  __device__ __forceinline__ unsigned int operator()(int u) const { return KEYS_IN_SMEM ? s_key[u] : compute(u); }
};

// the trie's levels 1..H (SidTrieLevels): each node's last code and its node in the level above
struct ExPath {
  const int* code[RQB_MAX_LEVELS + 1];
  const int* parent[RQB_MAX_LEVELS + 1];
};

template <bool KEYS_IN_SMEM, int FILTER>
__global__ void __launch_bounds__(RK_SEL_THREADS) t5exact_select_kernel(
    const float* __restrict__ sc, const int* __restrict__ coff, int n_root, const int* __restrict__ cnode,
    const long long* __restrict__ leaf_key, ExPath path, int H, int w, SidExcl f, int b0, int64_t* __restrict__ out_gen,
    float* __restrict__ out_lp) {
  using Scan = cub::BlockScan<int, RK_SEL_THREADS>;
  using Reduce = cub::BlockReduce<int, RK_SEL_THREADS>;
  __shared__ union {
    typename Scan::TempStorage scan;
    typename Reduce::TempStorage reduce;
  } tmp;
  __shared__ int hist[256];
  __shared__ int ctl[3];
  __shared__ int nsel_at, ties_base, n_valid;
  __shared__ unsigned long long sel[RK_SEL_MAX_N];
  extern __shared__ __align__(16) unsigned int s_key[];     // [U] when KEYS_IN_SMEM
  const int nt = RK_SEL_THREADS;
  const int b = blockIdx.x;
  const bool root = cnode == nullptr;
  const int64_t cs = root ? (int64_t)b * n_root : coff[b];
  const int U = root ? n_root : (int)(coff[b + 1] - cs);
  for (int i = threadIdx.x; i < 256; i += nt) hist[i] = 0;
  if (threadIdx.x == 0) {
    nsel_at = 0;
    ties_base = 0;
  }
  ExLeafKeys<KEYS_IN_SMEM, FILTER> key_of{s_key, sc + cs, root ? nullptr : cnode + cs, leaf_key, f, (int64_t)b0 + b, H};
  int mine = 0;
  for (int u = threadIdx.x; u < U; u += nt) {
    const unsigned int key = key_of.compute(u);
    if (KEYS_IN_SMEM) s_key[u] = key;
    mine += key != RK_BLOCKED;
  }
  const int valid = Reduce(tmp.reduce).Sum(mine);
  if (threadIdx.x == 0) n_valid = valid;
  __syncthreads();
  const int nsel = min(w, n_valid);
  unsigned int prefix, pmask;
  int want;
  rk_radix_threshold<true>(U, nsel, key_of, hist, ctl, prefix, pmask, want);
  // keep every candidate above the threshold and the `want` lowest-index ones at it (an ordered block scan over the ties)
  for (int base = 0; base < U; base += nt) {
    const int u = base + threadIdx.x;
    const unsigned int key = u < U ? key_of(u) : RK_BLOCKED;
    const bool in = nsel > 0 && key != RK_BLOCKED;
    const bool above = in && (key & pmask) > prefix;
    const int tie = (in && (key & pmask) == prefix) ? 1 : 0;
    int excl, total;
    Scan(tmp.scan).ExclusiveSum(tie, excl, total);
    if (above || (tie && ties_base + excl < want)) sel[atomicAdd(&nsel_at, 1)] = rk_key64(key, u);   // a slot only
    __syncthreads();                                        // scan storage and ties_base reused
    if (threadIdx.x == 0) ties_base += total;
    __syncthreads();
  }
  // each kept key's rank among the kept ones (distinct keys) is its output slot
  for (int i = threadIdx.x; i < nsel; i += nt) {
    const unsigned long long key = sel[i];
    int r = 0;
    for (int j = 0; j < nsel; ++j) r += sel[j] > key;
    const int u = (int)(0xffffffffu - (unsigned int)(key & 0xffffffffull));
    int node = root ? u : cnode[cs + u];                    // the leaf's tuple along its path
    int64_t* g = out_gen + ((int64_t)b * w + r) * H;
    for (int l = H; l >= 1; --l) {
      g[l - 1] = path.code[l][node];
      node = path.parent[l][node];
    }
    out_lp[(int64_t)b * w + r] = sc[cs + u];
  }
  for (int o = nsel + threadIdx.x; o < w; o += nt) {
    for (int h = 0; h < H; ++h) out_gen[((int64_t)b * w + o) * H + h] = -1;
    out_lp[(int64_t)b * w + o] = -INFINITY;
  }
}

static int ex_filter_of(const int* pos, const int64_t* keys, const int* count, int M, int H, int levels, bool include,
                        const char* what, SidExcl& f) {
  f = SidExcl{pos, reinterpret_cast<const long long*>(keys), count, M, H, include};
  RQB_CHECK_ARG(pos && keys && count && M > 0 && M <= SID_EXCL_MAX_M && H >= levels && H <= RQB_MAX_LEVELS,
                "%s: bad %s (M = %d, H = %d, need M <= %d and H >= %d)", what, include ? "inclusion" : "exclusion", M, H,
                SID_EXCL_MAX_M, levels);
  return RQB_OK;
}

template <bool WRITE, bool CAP>
static int ex_frontier_launch(int mode, dim3 grid, cudaStream_t st, const float* sc, const int* coff, int n_root, const int* cnode,
                              const int* ccode, const int* cpar, const int64_t* pkey, const float* tau, int Bc, int K, int l,
                              const int* lchild, const int* lcode_next, const SidExcl& f, int b0, int* counts, const int* offs,
                              int64_t* row_code, int64_t* row_par, float* row_score, int64_t* row_key, int* row_node, int* tiles,
                              int* nrng, int* nnode, int* ncode, int* npar, const ExCap& cap) {
  auto kernel = mode == SID_FILTER_INCLUDE   ? t5exact_frontier_kernel<SID_FILTER_INCLUDE, WRITE, CAP>
                : mode == SID_FILTER_EXCLUDE ? t5exact_frontier_kernel<SID_FILTER_EXCLUDE, WRITE, CAP>
                                             : t5exact_frontier_kernel<SID_FILTER_NONE, WRITE, CAP>;
  kernel<<<grid, EX_THREADS, 0, st>>>(sc, coff, n_root, cnode, ccode, cpar, reinterpret_cast<const long long*>(pkey), tau, Bc, K, l,
                                      lchild, lcode_next, f, b0, counts, offs, row_code, row_par, row_score,
                                      reinterpret_cast<long long*>(row_key), row_node, tiles, nrng, nnode, ncode, npar, cap);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

static int ex_frontier(int mode, const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode, const int* cpar,
                       const int64_t* pkey, const float* tau, int Bc, int K, int l, const int* lchild, const int* lcode_next, int b0,
                       int* counts, const int* offs, int64_t* row_code, int64_t* row_par, float* row_score, int64_t* row_key,
                       int* row_node, int* tiles, int* nrng, int* nnode, int* ncode, int* npar, const SidExcl& f, void* stream,
                       const ExCap* cap = nullptr) {
  RQB_CHECK_ARG(Bc >= 0 && K > 0 && l >= 1 && l < RQB_MAX_LEVELS && b0 >= 0 && n_root >= 0 && (counts != nullptr) != (offs != nullptr),
                "t5exact_frontier: bad argument (Bc = %d, K = %d, l = %d, b0 = %d; one of counts / offs)", Bc, K, l, b0);
  if (Bc == 0) return RQB_OK;
  RQB_CHECK_ARG(tau && lchild && ccode && (cnode ? coff && cpar && (mode == SID_FILTER_NONE || pkey) : l == 1),
                "t5exact_frontier: null pointer");
  RQB_CHECK_ARG(counts || (row_code && row_par && row_score && row_node && tiles && nrng && (mode == SID_FILTER_NONE || row_key)),
                "t5exact_frontier: null output");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (cap) {
    RQB_CHECK_ARG(offs && cap->r > 0 && cap->c > 0 && cap->t > 0, "t5exact_frontier_capacity: bad capacity (R = %d, C = %d, T = %d)",
                  cap->r, cap->c, cap->t);
    RQB_CHECK_ARG(cap->live && cap->overflow && cap->noff && nnode && ncode && npar, "t5exact_frontier_capacity: null output");
    return ex_frontier_launch<true, true>(mode, dim3(Bc), st, sc, coff, n_root, cnode, ccode, cpar, pkey, tau, Bc, K, l, lchild,
                                          lcode_next, f, b0, nullptr, offs, row_code, row_par, row_score, row_key, row_node, tiles, nrng,
                                          nnode, ncode, npar, *cap);
  }
  if (counts)
    return ex_frontier_launch<false, false>(mode, dim3(Bc), st, sc, coff, n_root, cnode, ccode, cpar, pkey, tau, Bc, K, l, lchild,
                                            lcode_next, f, b0, counts, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                                            nullptr, nullptr, nullptr, nullptr, ExCap{});
  return ex_frontier_launch<true, false>(mode, dim3(Bc), st, sc, coff, n_root, cnode, ccode, cpar, pkey, tau, Bc, K, l, lchild,
                                         lcode_next, f, b0, nullptr, offs, row_code, row_par, row_score, row_key, row_node, tiles, nrng,
                                         nnode, ncode, npar, ExCap{});
}

extern "C" int rqb200_t5exact_frontier(const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode,
                                       const int* cpar, const int64_t* pkey, const float* tau, int Bc, int K, int l, const int* lchild,
                                       const int* lcode_next, int b0, int* counts, const int* offs, int64_t* row_code,
                                       int64_t* row_par, float* row_score, int64_t* row_key, int* row_node, int* tiles, int* nrng,
                                       int* nnode, int* ncode, int* npar, void* stream) {
  return ex_frontier(SID_FILTER_NONE, sc, coff, n_root, cnode, ccode, cpar, pkey, tau, Bc, K, l, lchild, lcode_next, b0, counts, offs,
                     row_code, row_par, row_score, row_key, row_node, tiles, nrng, nnode, ncode, npar, SidExcl{}, stream);
}

#define EX_FRONTIER_FILTERED(NAME, MODE, INCLUDE)                                                                                    \
  extern "C" int NAME(const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode, const int* cpar,             \
                      const int64_t* pkey, const float* tau, int Bc, int K, int l, const int* lchild, const int* lcode_next, int b0, \
                      int* counts, const int* offs, int64_t* row_code, int64_t* row_par, float* row_score, int64_t* row_key,       \
                      int* row_node, int* tiles, int* nrng, int* nnode, int* ncode, int* npar, const int* f_pos,                  \
                      const int64_t* f_keys, const int* f_count, int f_M, int f_H, void* stream) {                                 \
    SidExcl f;                                                                                                                      \
    const int rc = ex_filter_of(f_pos, f_keys, f_count, f_M, f_H, l, INCLUDE, #NAME, f);                                            \
    if (rc != RQB_OK) return rc;                                                                                                    \
    return ex_frontier(MODE, sc, coff, n_root, cnode, ccode, cpar, pkey, tau, Bc, K, l, lchild, lcode_next, b0, counts, offs,       \
                       row_code, row_par, row_score, row_key, row_node, tiles, nrng, nnode, ncode, npar, f, stream);                \
  }
EX_FRONTIER_FILTERED(rqb200_t5exact_frontier_excluding, SID_FILTER_EXCLUDE, false)
EX_FRONTIER_FILTERED(rqb200_t5exact_frontier_including, SID_FILTER_INCLUDE, true)

// the write pass at fixed capacities (ExCap): offs as the write pass's, the totals read on the device
extern "C" int rqb200_t5exact_frontier_capacity(const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode,
                                                const int* cpar, const int64_t* pkey, const float* tau, int Bc, int K, int l,
                                                const int* lchild, const int* lcode_next, int b0, const int* offs, int64_t* row_code,
                                                int64_t* row_par, float* row_score, int64_t* row_key, int* row_node, int* tiles,
                                                int* nrng, int* nnode, int* ncode, int* npar, int r_cap, int c_cap, int t_cap,
                                                int* live, int* overflow, int* noff, void* stream) {
  const ExCap cap{r_cap, c_cap, t_cap, live, overflow, noff};
  return ex_frontier(SID_FILTER_NONE, sc, coff, n_root, cnode, ccode, cpar, pkey, tau, Bc, K, l, lchild, lcode_next, b0, nullptr, offs,
                     row_code, row_par, row_score, row_key, row_node, tiles, nrng, nnode, ncode, npar, SidExcl{}, stream, &cap);
}

#define EX_FRONTIER_CAPACITY_FILTERED(NAME, MODE, INCLUDE)                                                                           \
  extern "C" int NAME(const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode, const int* cpar,             \
                      const int64_t* pkey, const float* tau, int Bc, int K, int l, const int* lchild, const int* lcode_next, int b0, \
                      const int* offs, int64_t* row_code, int64_t* row_par, float* row_score, int64_t* row_key, int* row_node,     \
                      int* tiles, int* nrng, int* nnode, int* ncode, int* npar, int r_cap, int c_cap, int t_cap, int* live,        \
                      int* overflow, int* noff, const int* f_pos, const int64_t* f_keys, const int* f_count, int f_M, int f_H,     \
                      void* stream) {                                                                                               \
    SidExcl f;                                                                                                                      \
    const int rc = ex_filter_of(f_pos, f_keys, f_count, f_M, f_H, l, INCLUDE, #NAME, f);                                            \
    if (rc != RQB_OK) return rc;                                                                                                    \
    const ExCap cap{r_cap, c_cap, t_cap, live, overflow, noff};                                                                     \
    return ex_frontier(MODE, sc, coff, n_root, cnode, ccode, cpar, pkey, tau, Bc, K, l, lchild, lcode_next, b0, nullptr, offs,      \
                       row_code, row_par, row_score, row_key, row_node, tiles, nrng, nnode, ncode, npar, f, stream, &cap);          \
  }
EX_FRONTIER_CAPACITY_FILTERED(rqb200_t5exact_frontier_capacity_excluding, SID_FILTER_EXCLUDE, false)
EX_FRONTIER_CAPACITY_FILTERED(rqb200_t5exact_frontier_capacity_including, SID_FILTER_INCLUDE, true)

template <bool KEYS_IN_SMEM>
static int ex_select_launch(int mode, int Bc, size_t smem, cudaStream_t st, const float* sc, const int* coff, int n_root,
                            const int* cnode, const int64_t* leaf_key, const ExPath& path, int H, int w, const SidExcl& f, int b0,
                            int64_t* out_gen, float* out_lp) {
  auto kernel = mode == SID_FILTER_INCLUDE   ? t5exact_select_kernel<KEYS_IN_SMEM, SID_FILTER_INCLUDE>
                : mode == SID_FILTER_EXCLUDE ? t5exact_select_kernel<KEYS_IN_SMEM, SID_FILTER_EXCLUDE>
                                             : t5exact_select_kernel<KEYS_IN_SMEM, SID_FILTER_NONE>;
  if (KEYS_IN_SMEM) {
    static unsigned long long done[3] = {0, 0, 0};
    const int rc = rk_set_smem_once(reinterpret_cast<const void*>(kernel), RK_SEL_SMEM_KEYS * (int)sizeof(unsigned int), &done[mode]);
    if (rc != RQB_OK) return rc;
  }
  kernel<<<Bc, RK_SEL_THREADS, smem, st>>>(sc, coff, n_root, cnode, reinterpret_cast<const long long*>(leaf_key), path, H, w, f, b0,
                                           out_gen, out_lp);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

static int ex_select(int mode, const float* sc, const int* coff, int n_root, const int* cnode, int max_u, const int64_t* leaf_key,
                     const void* const* codes, const void* const* parents, int Bc, int H, int w, int b0, int64_t* out_gen,
                     float* out_lp, const SidExcl& f, void* stream) {
  RQB_CHECK_ARG(Bc >= 0 && H > 0 && w > 0 && b0 >= 0 && n_root >= 0 && max_u >= 0,
                "t5exact_select: bad argument (Bc = %d, H = %d, w = %d, b0 = %d)", Bc, H, w, b0);
  if (w > RK_SEL_MAX_N || H > RQB_MAX_LEVELS) {
    rqb_set_error("t5exact_select: need w <= %d and H <= %d (w = %d, H = %d)", RK_SEL_MAX_N, RQB_MAX_LEVELS, w, H);
    return RQB_ERR_UNSUPPORTED;
  }
  if (Bc == 0) return RQB_OK;
  RQB_CHECK_ARG((sc || max_u == 0) && (cnode ? coff != nullptr : true) && (leaf_key || mode == SID_FILTER_NONE) && codes &&
                    parents && out_gen && out_lp,
                "t5exact_select: null pointer");
  ExPath path{};
  for (int l = 1; l <= H; ++l) {
    path.code[l] = static_cast<const int*>(codes[l]);
    path.parent[l] = static_cast<const int*>(parents[l]);
    RQB_CHECK_ARG(max_u == 0 || (path.code[l] && path.parent[l]), "t5exact_select: null level %d", l);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (max_u <= RK_SEL_SMEM_KEYS)
    return ex_select_launch<true>(mode, Bc, (size_t)max_u * sizeof(unsigned int), st, sc, coff, n_root, cnode, leaf_key, path, H,
                                  w, f, b0, out_gen, out_lp);
  return ex_select_launch<false>(mode, Bc, 0, st, sc, coff, n_root, cnode, leaf_key, path, H, w, f, b0, out_gen, out_lp);
}

extern "C" int rqb200_t5exact_select(const float* sc, const int* coff, int n_root, const int* cnode, int max_u,
                                     const int64_t* leaf_key, const void* const* codes, const void* const* parents, int Bc, int H,
                                     int w, int b0, int64_t* out_gen, float* out_lp, void* stream) {
  return ex_select(SID_FILTER_NONE, sc, coff, n_root, cnode, max_u, leaf_key, codes, parents, Bc, H, w, b0, out_gen, out_lp,
                   SidExcl{}, stream);
}

#define EX_SELECT_FILTERED(NAME, MODE, INCLUDE)                                                                                      \
  extern "C" int NAME(const float* sc, const int* coff, int n_root, const int* cnode, int max_u, const int64_t* leaf_key,          \
                      const void* const* codes, const void* const* parents, int Bc, int H, int w, int b0, int64_t* out_gen,      \
                      float* out_lp, const int* f_pos, const int64_t* f_keys, const int* f_count, int f_M, int f_H,              \
                      void* stream) {                                                                                               \
    SidExcl f;                                                                                                                      \
    const int rc = ex_filter_of(f_pos, f_keys, f_count, f_M, f_H, H, INCLUDE, #NAME, f);                                            \
    if (rc != RQB_OK) return rc;                                                                                                    \
    return ex_select(MODE, sc, coff, n_root, cnode, max_u, leaf_key, codes, parents, Bc, H, w, b0, out_gen, out_lp, f, stream);   \
  }
EX_SELECT_FILTERED(rqb200_t5exact_select_excluding, SID_FILTER_EXCLUDE, false)
EX_SELECT_FILTERED(rqb200_t5exact_select_including, SID_FILTER_INCLUDE, true)
