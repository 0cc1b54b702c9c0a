// TF32 tensor-core self-attention of the packed T5 encoder pass (generate / forward with encoder="fused",
// encoder_attention="tf32").  Same inputs, outputs and conventions as rqb200_t5enc_attention, _attention_train and
// _attention_backward of csrc/t5enc.cu: qkv [N, 3 inner] packed rows, history b owns rows offsets[b] .. offsets[b + 1] - 1,
// scores q . k + (rel[pj - pi] + key_mask) with no 1/sqrt(d) scaling, lse = (m - key_mask) + log l, the same Philox keep bits
// (csrc/t5_dropout.cuh), no global atomics.  What changes is the precision of the four kinds of products (scores, P.V, dP and
// the gradient products): they run as wgmma m64n64k8 TF32 with fp32 accumulation, the operands rounded to TF32 (cvt.rna) as
// they are staged.  Softmax, bias, mask, dropout and D = rowsum(dO o O) stay fp32.
//
//   rqb200_t5enc_attention_tc[_train]  one warpgroup per (history, head, 64-query tile): S = Q K^T from shared memory, online
//                                      softmax in registers, O += P V with P as the register A operand.
//   rqb200_t5enc_attention_tc_backward a query-major launch (D, dQ += dS K, the per-CTA partials of d_rel) and a key-major launch
//                                      (S^T = K Q^T, dV += P^T dO, dK += dS^T Q).
//
// Shared-memory operands use wgmma's K-major layout without swizzle: 8 x 4 fp32 core matrices of 128 contiguous bytes, the
// cores of one 8-row group side by side along K (LBO 128 B), 8-row groups 2048 B apart (SBO).  TF32 wgmma reads shared memory
// only K-major, so every B operand whose contraction runs over rows of qkv / dout (V for P V, K for dS K, dO and Q for the dV / dK
// products) is staged by a transposing copy.  That copy also permutes the keys of each group of 8 to 0,2,4,6,1,3,5,7: an
// accumulator thread holds columns 2t and 2t + 1 of an 8-column block, the TF32 A fragment wants columns t and t + 4, and the
// permutation makes the accumulator registers the A fragment as they are.
//
// d_rel: the query-major CTA copies each dS tile to shared memory and adds it into two shared bin arrays of 2S - 1 floats, one
// per half of the tile's queries.  In a round, the 64 threads of a half each add one key column of one query row; the columns
// of one row have distinct positions, so they hit distinct bins, and a named barrier orders the rounds: a fixed summation order,
// bit-reproducible, in 32 rounds per tile for each half.  The bins take 2 (2S - 1) floats, 80 KB at S = 5120, next to 97 KB of
// tiles; one bin array per warp would not fit there.
#include <cfloat>

#include "common.cuh"
#include "t5_dropout.cuh"
#include "t5_tc.cuh"

extern __shared__ __align__(128) float tc_smem[];

// ------------------------------------------------------------------------------------------------ forward
// grid (B, heads, ceil(S / 64)), 128 threads, dynamic smem 3 tiles + 64 ints.  Thread (warp w, lane 4 g + t) holds the rows
// 16 w + g and 16 w + g + 8 of the query tile and, of each 8-key block j, columns 8 j + 2 t and 8 j + 2 t + 1.
template <bool TRAIN>
__global__ void __launch_bounds__(TC_THREADS) t5tc_attention_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, const int* __restrict__ src, const int* __restrict__ offsets,
    const float* __restrict__ key_mask, const float* __restrict__ rel, int S, int heads, float* __restrict__ out, int64_t ldo,
    const int64_t* __restrict__ seed, uint32_t thresh, float scale, float* __restrict__ lse) {
  float* sQ = tc_smem;
  float* sK = sQ + TC_TILE;
  float* sVt = sK + TC_TILE;
  int* spos = reinterpret_cast<int*>(sVt + TC_TILE);
  const int b = blockIdx.x, n = blockIdx.y;
  const int off = offsets[b], cnt = offsets[b + 1] - off;
  const int q0 = blockIdx.z * TC_T;
  if (q0 >= cnt) return;                                      // uniform over the CTA
  const int nq = min(TC_T, cnt - q0);
  const int64_t inner = (int64_t)heads * 64;
  const float km = key_mask[b];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int row[2] = {16 * warp + g, 16 * warp + g + 8};
  const bool act[2] = {row[0] < nq, row[1] < nq};
  int pi[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) pi[h] = act[h] ? src[off + q0 + row[h]] - b * S : 0;
  const float* relh = rel + (int64_t)n * (2 * S - 1) + (S - 1);
  tc_stage(sQ, qkv + (int64_t)(off + q0) * ldqkv + n * 64, ldqkv, nq);

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint2 key = TRAIN && thresh ? te_seed_key(seed) : make_uint2(0u, 0u);

  for (int t0 = 0; t0 < cnt; t0 += TC_T) {
    const int nk = min(TC_T, cnt - t0);
    __syncthreads();                                          // the previous tile's MMAs have completed in every warp
    const float* kv = qkv + (int64_t)(off + t0) * ldqkv + n * 64;
    tc_stage(sK, kv + inner, ldqkv, nk);
    tc_stage_t(sVt, kv + 2 * inner, ldqkv, nk);
    if (threadIdx.x < TC_T) spos[threadIdx.x] = (int)threadIdx.x < nk ? src[off + t0 + threadIdx.x] - b * S : -1;
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
        const int pj = spos[8 * j + 2 * t + e];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float& v = s[4 * j + 2 * h + e];
          v = pj < 0 ? -INFINITY : v + (relh[pj - pi[h]] + km);   // a key past the history contributes exp(-inf) = 0
          mt[h] = fmaxf(mt[h], v);
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
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int pj = spos[8 * j + 2 * t + e];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = 4 * j + 2 * h + e;
          float p = expf(s[i] - m[h]);
          lt[h] += p;
          if (TRAIN && thresh && act[h] && pj >= 0 && !te_keep(key, b, n, pi[h], pj, thresh)) p = 0.f;
          a[i] = tf32_bits(p);
        }
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
    if (!act[h]) continue;
    const int64_t r = off + q0 + row[h];
    float* orow = out + r * ldo + n * 64 + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float2 v = make_float2(o[4 * j + 2 * h] / l[h], o[4 * j + 2 * h + 1] / l[h]);
      if (TRAIN && thresh) v = make_float2(v.x * scale, v.y * scale);
      *reinterpret_cast<float2*>(orow + 8 * j) = v;
    }
    if (TRAIN && t == 0) lse[r * heads + n] = (m[h] - km) + logf(l[h]);
  }
}

// ------------------------------------------------------------------------------------------------ backward, query-major
// dS_ij = P_ij (dP_ij z_ij - D_i), z_ij = keep_ij * scale, dP_ij = dO_i . v_j, D_i = dO_i . O_i, P_ij = exp((s_ij - key_mask) - lse_i).
#define TC_DS_LD 65              // row stride of the shared dS copy (conflict-free column reads)
static size_t tc_bwd_q_smem(int S) {
  return (5 * TC_TILE + TC_T * TC_DS_LD + 2 * TC_T + 2 * (2 * (size_t)S - 1)) * sizeof(float);
}

// grid (B, heads, ceil(S / 64)), 128 threads.  Writes delta [N, heads], dQ into dqkv and drel_part[((b * tiles + z) * heads + n)
// * (2S - 1) + t] (zeros for a tile past the history).
__global__ void __launch_bounds__(TC_THREADS) t5tc_attention_bwd_q_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, const float* __restrict__ o, int64_t ldo, const float* __restrict__ dout,
    int64_t lddo, const float* __restrict__ lse, const int* __restrict__ src, const int* __restrict__ offsets,
    const float* __restrict__ key_mask, const float* __restrict__ rel, int S, int heads, const int64_t* __restrict__ seed,
    uint32_t thresh, float scale, float* __restrict__ delta, float* __restrict__ dqkv, int64_t ldd, float* __restrict__ drel_part) {
  const int R = 2 * S - 1;
  float* sQ = tc_smem;
  float* sdO = sQ + TC_TILE;
  float* sK = sdO + TC_TILE;
  float* sKt = sK + TC_TILE;
  float* sV = sKt + TC_TILE;
  float* sdS = sV + TC_TILE;                                  // [64][TC_DS_LD]
  int* sqpos = reinterpret_cast<int*>(sdS + TC_T * TC_DS_LD);
  int* spos = sqpos + TC_T;
  float* bins = reinterpret_cast<float*>(spos + TC_T);        // [2][R]: queries 0 .. 31 and 32 .. 63
  const int b = blockIdx.x, n = blockIdx.y;
  const int off = offsets[b], cnt = offsets[b + 1] - off;
  const int q0 = blockIdx.z * TC_T;
  float* part = drel_part + (((int64_t)b * gridDim.z + blockIdx.z) * heads + n) * R;
  if (q0 >= cnt) {                                            // uniform over the CTA
    for (int i = threadIdx.x; i < R; i += TC_THREADS) part[i] = 0.f;
    return;
  }
  const int nq = min(TC_T, cnt - q0);
  const int64_t inner = (int64_t)heads * 64;
  const float km = key_mask[b];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int row[2] = {16 * warp + g, 16 * warp + g + 8};
  const bool act[2] = {row[0] < nq, row[1] < nq};

  tc_stage(sQ, qkv + (int64_t)(off + q0) * ldqkv + n * 64, ldqkv, nq);
  tc_stage(sdO, dout + (int64_t)(off + q0) * lddo + n * 64, lddo, nq);
  {                                                           // D_i: two threads per query, 32 dimensions each
    const int i = threadIdx.x >> 1, hh = threadIdx.x & 1;
    float di = 0.f;
    if (i < nq) {
      const float4* gr = reinterpret_cast<const float4*>(dout + (int64_t)(off + q0 + i) * lddo + n * 64) + hh * 8;
      const float4* orw = reinterpret_cast<const float4*>(o + (int64_t)(off + q0 + i) * ldo + n * 64) + hh * 8;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float4 gc = gr[c], oc = orw[c];
        di = fmaf(gc.x, oc.x, di);
        di = fmaf(gc.y, oc.y, di);
        di = fmaf(gc.z, oc.z, di);
        di = fmaf(gc.w, oc.w, di);
      }
    }
    di += __shfl_xor_sync(0xffffffffu, di, 1);
    if (i < nq && hh == 0) {
      delta[(int64_t)(off + q0 + i) * heads + n] = di;
      sdS[i] = di;                                            // parked here until the first tile
    }
  }
  if (threadIdx.x < TC_T) sqpos[threadIdx.x] = (int)threadIdx.x < nq ? src[off + q0 + threadIdx.x] - b * S : -1;
  for (int i = threadIdx.x; i < 2 * R; i += TC_THREADS) bins[i] = 0.f;
  __syncthreads();
  float di[2], li[2];
  int pi[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    di[h] = act[h] ? sdS[row[h]] : 0.f;
    li[h] = act[h] ? lse[(int64_t)(off + q0 + row[h]) * heads + n] : 0.f;
    pi[h] = act[h] ? sqpos[row[h]] : 0;
  }
  const float* relh = rel + (int64_t)n * R + (S - 1);
  const uint2 key = thresh ? te_seed_key(seed) : make_uint2(0u, 0u);
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  const int half = threadIdx.x >> 6, col = threadIdx.x & 63;  // the d_rel rounds: queries 32 half .., key column col
  float* hbins = bins + half * R + (S - 1);

  for (int t0 = 0; t0 < cnt; t0 += TC_T) {
    const int nk = min(TC_T, cnt - t0);
    __syncthreads();                                          // the previous tile is consumed (MMAs, dS copy, rounds)
    const float* kv = qkv + (int64_t)(off + t0) * ldqkv + n * 64;
    tc_stage(sK, kv + inner, ldqkv, nk);
    tc_stage_t(sKt, kv + inner, ldqkv, nk);
    tc_stage(sV, kv + 2 * inner, ldqkv, nk);
    if (threadIdx.x < TC_T) spos[threadIdx.x] = (int)threadIdx.x < nk ? src[off + t0 + threadIdx.x] - b * S : -1;
    tc_proxy_fence();
    __syncthreads();
    float s[32], dp[32];
    tc_fence();
    tc_gemm_ss(s, sQ, sK);
    tc_gemm_ss(dp, sdO, sV);
    tc_commit();
    tc_wait();
    tc_pin(s);
    tc_pin(dp);
    uint32_t a[32];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = 8 * j + 2 * t + e, pj = spos[c];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = 4 * j + 2 * h + e;
          float ds = 0.f;
          if (act[h] && pj >= 0) {
            const float sc = s[i] + (relh[pj - pi[h]] + km);
            const float p = expf((sc - km) - li[h]);
            const float z = thresh ? (te_keep(key, b, n, pi[h], pj, thresh) ? scale : 0.f) : 1.f;
            ds = p * (dp[i] * z - di[h]);
          }
          sdS[row[h] * TC_DS_LD + c] = ds;
          a[i] = tf32_bits(ds);
        }
      }
    tc_fence();
    tc_gemm_rs(dq, a, sKt);
    tc_commit();
    __syncthreads();                                          // the dS copy is complete
    const int pj = spos[col];
    for (int i = 32 * half; i < 32 * half + 32; ++i) {
      const int p = sqpos[i];
      if (pj >= 0 && p >= 0) hbins[pj - p] += sdS[i * TC_DS_LD + col];   // one query's 64 columns hit 64 distinct bins
      asm volatile("bar.sync %0, 64;" ::"r"(1 + half) : "memory");
    }
    tc_wait();
    tc_pin(dq);
    tc_pin(a);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!act[h]) continue;
    float* dr = dqkv + (int64_t)(off + q0 + row[h]) * ldd + n * 64 + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) *reinterpret_cast<float2*>(dr + 8 * j) = make_float2(dq[4 * j + 2 * h], dq[4 * j + 2 * h + 1]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < R; i += TC_THREADS) part[i] = bins[i] + bins[R + i];
}

// ------------------------------------------------------------------------------------------------ backward, key-major
// grid (B, heads, ceil(S / 64)), 128 threads: S^T = K Q^T and dP^T = V dO^T per query tile, dV += (P z)^T dO and dK += dS^T Q.
__global__ void __launch_bounds__(TC_THREADS) t5tc_attention_bwd_kv_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, const float* __restrict__ dout, int64_t lddo, const float* __restrict__ lse,
    const float* __restrict__ delta, const int* __restrict__ src, const int* __restrict__ offsets,
    const float* __restrict__ key_mask, const float* __restrict__ rel, int S, int heads, const int64_t* __restrict__ seed,
    uint32_t thresh, float scale, float* __restrict__ dqkv, int64_t ldd) {
  float* sK = tc_smem;
  float* sV = sK + TC_TILE;
  float* sQ = sV + TC_TILE;
  float* sdO = sQ + TC_TILE;
  float* sQt = sdO + TC_TILE;
  float* sdOt = sQt + TC_TILE;
  float* slse = sdOt + TC_TILE;
  float* sd = slse + TC_T;
  int* sqpos = reinterpret_cast<int*>(sd + TC_T);
  const int b = blockIdx.x, n = blockIdx.y;
  const int off = offsets[b], cnt = offsets[b + 1] - off;
  const int k0 = blockIdx.z * TC_T;
  if (k0 >= cnt) return;                                      // uniform over the CTA
  const int nk = min(TC_T, cnt - k0);
  const int64_t inner = (int64_t)heads * 64;
  const float km = key_mask[b];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int row[2] = {16 * warp + g, 16 * warp + g + 8};
  const bool act[2] = {row[0] < nk, row[1] < nk};
  int pj[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) pj[h] = act[h] ? src[off + k0 + row[h]] - b * S : 0;
  const float* kvb = qkv + (int64_t)(off + k0) * ldqkv + n * 64;
  tc_stage(sK, kvb + inner, ldqkv, nk);
  tc_stage(sV, kvb + 2 * inner, ldqkv, nk);
  const float* relh = rel + (int64_t)n * (2 * S - 1) + (S - 1);
  const uint2 key = thresh ? te_seed_key(seed) : make_uint2(0u, 0u);
  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dk[i] = dv[i] = 0.f;

  for (int t0 = 0; t0 < cnt; t0 += TC_T) {
    const int nq = min(TC_T, cnt - t0);
    __syncthreads();
    const float* qb = qkv + (int64_t)(off + t0) * ldqkv + n * 64;
    const float* gb = dout + (int64_t)(off + t0) * lddo + n * 64;
    tc_stage(sQ, qb, ldqkv, nq);
    tc_stage(sdO, gb, lddo, nq);
    tc_stage_t(sQt, qb, ldqkv, nq);
    tc_stage_t(sdOt, gb, lddo, nq);
    if (threadIdx.x < TC_T) {
      const int i = t0 + threadIdx.x;
      const bool in = (int)threadIdx.x < nq;
      sqpos[threadIdx.x] = in ? src[off + i] - b * S : -1;
      slse[threadIdx.x] = in ? lse[(int64_t)(off + i) * heads + n] : 0.f;
      sd[threadIdx.x] = in ? delta[(int64_t)(off + i) * heads + n] : 0.f;
    }
    tc_proxy_fence();
    __syncthreads();
    float s[32], dp[32];
    tc_fence();
    tc_gemm_ss(s, sK, sQ);
    tc_gemm_ss(dp, sV, sdO);
    tc_commit();
    tc_wait();
    tc_pin(s);
    tc_pin(dp);
    uint32_t apz[32], ads[32];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = 8 * j + 2 * t + e, pi = sqpos[c];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = 4 * j + 2 * h + e;
          float pz = 0.f, ds = 0.f;
          if (act[h] && pi >= 0) {
            const float sc = s[i] + (relh[pj[h] - pi] + km);
            const float p = expf((sc - km) - slse[c]);
            const float z = thresh ? (te_keep(key, b, n, pi, pj[h], thresh) ? scale : 0.f) : 1.f;
            pz = p * z;
            ds = p * (dp[i] * z - sd[c]);
          }
          apz[i] = tf32_bits(pz);
          ads[i] = tf32_bits(ds);
        }
      }
    tc_fence();
    tc_gemm_rs(dv, apz, sdOt);
    tc_gemm_rs(dk, ads, sQt);
    tc_commit();
    tc_wait();
    tc_pin(dv);
    tc_pin(dk);
    tc_pin(apz);
    tc_pin(ads);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!act[h]) continue;
    float* dr = dqkv + (int64_t)(off + k0 + row[h]) * ldd + n * 64 + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<float2*>(dr + inner + 8 * j) = make_float2(dk[4 * j + 2 * h], dk[4 * j + 2 * h + 1]);
      *reinterpret_cast<float2*>(dr + 2 * inner + 8 * j) = make_float2(dv[4 * j + 2 * h], dv[4 * j + 2 * h + 1]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ C ABI
#define TC_FWD_SMEM (3 * TC_TILE * sizeof(float) + TC_T * sizeof(int))
#define TC_KV_SMEM ((6 * TC_TILE + 3 * TC_T) * sizeof(float))
#define TC_SMEM_MAX (227 * 1024)

static int tc_args(const float* qkv, int64_t ldqkv, int B, int S, int heads, float p, const char* what) {
  RQB_CHECK_ARG(B >= 0 && S > 0 && heads > 0, "%s: bad shape (B=%d S=%d heads=%d)", what, B, S, heads);
  RQB_CHECK_ARG(p >= 0.f && p < 1.f, "%s: dropout probability %g outside [0, 1)", what, (double)p);
  RQB_CHECK_ARG(ldqkv >= 3 * (int64_t)heads * 64 && ldqkv % 4 == 0 && reinterpret_cast<uintptr_t>(qkv) % 16 == 0,
                "%s: qkv needs a row stride >= 3 * heads * 64 that is a multiple of 4 and 16-byte alignment", what);
  RQB_CHECK_ARG(heads <= 65535 && (int64_t)B * S <= INT32_MAX, "%s: too many heads or positions", what);
  return RQB_OK;
}

static int tc_forward(const float* qkv, int64_t ldqkv, const int* src, const int* offsets, const float* key_mask, const float* rel,
                      int B, int S, int heads, const int64_t* seed, float p, float* out, int64_t ldo, float* lse, bool train,
                      void* stream, const char* what) {
  if (int rc = tc_args(qkv, ldqkv, B, S, heads, p, what)) return rc;
  RQB_CHECK_ARG(ldo >= (int64_t)heads * 64 && ldo % 4 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0,
                "%s: out needs a row stride >= heads * 64 that is a multiple of 4 and 16-byte alignment", what);
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(qkv && src && offsets && key_mask && rel && out && (!train || (lse && seed)), "%s: null pointer", what);
  uint32_t thresh = 0;
  float scale = 1.f;
  if (train) dropout_params(p, &thresh, &scale);
  const dim3 grid(B, heads, (unsigned)((S + TC_T - 1) / TC_T));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (train) {
    RQB_CUDA(cudaFuncSetAttribute(t5tc_attention_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_FWD_SMEM));
    t5tc_attention_kernel<true><<<grid, TC_THREADS, TC_FWD_SMEM, st>>>(qkv, ldqkv, src, offsets, key_mask, rel, S, heads, out, ldo,
                                                                        seed, thresh, scale, lse);
  } else {
    RQB_CUDA(cudaFuncSetAttribute(t5tc_attention_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_FWD_SMEM));
    t5tc_attention_kernel<false><<<grid, TC_THREADS, TC_FWD_SMEM, st>>>(qkv, ldqkv, src, offsets, key_mask, rel, S, heads, out,
                                                                         ldo, nullptr, 0u, 1.f, nullptr);
  }
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5enc_attention_tc(const float* qkv, int64_t ldqkv, const int* src, const int* offsets, const float* key_mask,
                                         const float* rel, int B, int S, int heads, float* out, int64_t ldo, void* stream) {
  return tc_forward(qkv, ldqkv, src, offsets, key_mask, rel, B, S, heads, nullptr, 0.f, out, ldo, nullptr, false, stream,
                    "t5enc_attention_tc");
}

extern "C" int rqb200_t5enc_attention_tc_train(const float* qkv, int64_t ldqkv, const int* src, const int* offsets,
                                               const float* key_mask, const float* rel, int B, int S, int heads,
                                               const int64_t* seed, float p, float* out, int64_t ldo, float* lse, void* stream) {
  return tc_forward(qkv, ldqkv, src, offsets, key_mask, rel, B, S, heads, seed, p, out, ldo, lse, true, stream,
                    "t5enc_attention_tc_train");
}

extern "C" int rqb200_t5enc_attention_tc_backward_tiles(int S) { return S > 0 ? (S + TC_T - 1) / TC_T : 0; }

extern "C" int rqb200_t5enc_attention_tc_backward(const float* qkv, int64_t ldqkv, const float* out, int64_t ldo,
                                                  const float* dout, int64_t lddo, const float* lse, const int* src,
                                                  const int* offsets, const float* key_mask, const float* rel, int B, int S,
                                                  int heads, const int64_t* seed, float p, float* delta, float* dqkv, int64_t ldd,
                                                  float* drel_part, void* stream) {
  if (int rc = tc_args(qkv, ldqkv, B, S, heads, p, "t5enc_attention_tc_backward")) return rc;
  const int64_t inner = (int64_t)heads * 64;
  RQB_CHECK_ARG(ldo >= inner && lddo >= inner && ldd >= 3 * inner && ldo % 4 == 0 && lddo % 4 == 0 && ldd % 4 == 0 &&
                    ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(dout) | reinterpret_cast<uintptr_t>(dqkv)) %
                     16) == 0,
                "t5enc_attention_tc_backward: out / dout need row strides >= heads * 64, dqkv >= 3 * heads * 64, all multiples "
                "of 4, and 16-byte alignment");
  const size_t smem = tc_bwd_q_smem(S);
  RQB_CHECK_ARG(smem <= TC_SMEM_MAX, "t5enc_attention_tc_backward: S = %d positions exceed the relative-bias bins' shared "
                "memory (at most %d)", S, (int)((TC_SMEM_MAX - tc_bwd_q_smem(1)) / (4 * sizeof(float))) + 1);
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(qkv && out && dout && lse && src && offsets && key_mask && rel && seed && delta && dqkv && drel_part,
                "t5enc_attention_tc_backward: null pointer");
  uint32_t thresh;
  float scale;
  dropout_params(p, &thresh, &scale);
  const dim3 grid(B, heads, (unsigned)rqb200_t5enc_attention_tc_backward_tiles(S));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RQB_CUDA(cudaFuncSetAttribute(t5tc_attention_bwd_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  t5tc_attention_bwd_q_kernel<<<grid, TC_THREADS, smem, st>>>(qkv, ldqkv, out, ldo, dout, lddo, lse, src, offsets, key_mask, rel,
                                                              S, heads, seed, thresh, scale, delta, dqkv, ldd, drel_part);
  RQB_LAUNCH_CHECK();
  RQB_CUDA(cudaFuncSetAttribute(t5tc_attention_bwd_kv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_KV_SMEM));
  t5tc_attention_bwd_kv_kernel<<<grid, TC_THREADS, TC_KV_SMEM, st>>>(qkv, ldqkv, dout, lddo, lse, delta, src, offsets, key_mask,
                                                                     rel, S, heads, seed, thresh, scale, dqkv, ldd);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}
