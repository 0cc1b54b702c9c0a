// One decoder step of the generative-retrieval model's T5 stack (transformers T5Stack in eval mode, is_decoder=True) for the
// fused decode path of EncoderDecoderRetrievalModel.generate(decoder="fused").  The GEMMs stay with cuBLAS; these kernels do
// what lies between them, without copying any key/value state:
//
//   rqb200_t5dec_cross_attention  attention over the encoder output, one CTA per (history, head).  Every beam of a history has the
//                                 same cross keys and values, so they are stored once per history ([B, S] rows) and the CTA reads
//                                 them once for up to 32 of the history's nq queries (1 at level 0, the beam width later).  Keys stream through
//                                 shared memory 32 at a time with an online softmax: the encoder length has no fixed limit.
//   rqb200_t5dec_self_attention   the step's causal self-attention, one warp per (beam row, head).  The step's own key/value go to
//                                 slot h of a cache of H positions; earlier positions are read through an int32 ancestor table
//                                 [rows, H] (the row of each earlier level this beam descends from), so a reordered beam never
//                                 copies its past.  With `parent` the kernel also advances the table: anc_out[r] = anc_in[parent[r]]
//                                 with position h - 1 set to parent[r].
//   rqb200_t5dec_add_norm         a sublayer boundary, one warp per row: x += delta (or x = the step's input embedding), then
//                                 out = T5LayerNorm(x) * weight.
//
// Numerics are HF's: attention without 1/sqrt(d) scaling, fp32 softmax, masked encoder keys get -FLT_MAX added
// (torch.finfo(float32).min, as HF's eager mask does: a history with no unmasked key averages all its values), RMS norm in fp32.
//
// The training pass (forward(decoder="fused")) runs T <= 8 decoder positions per history, rows b * T + t, and adds:
//   rqb200_t5dec_self_attention_train / _backward    causal self-attention, one warp per (history, head) with the history's keys
//                                                    and values in registers.  The forward applies HF's attention-weight dropout
//                                                    and saves the log-sum-exp; the backward recomputes P and writes dQ, dK, dV
//                                                    and per-warp partials of the [heads, 2T - 1] relative-bias gradient.
//   rqb200_t5dec_cross_attention_train / _backward   attention over encoder rows laid out by offsets (history b's keys are rows
//                                                    offsets[b] .. offsets[b + 1] - 1: packed kept rows or [B * S] padded rows)
//                                                    with an additive per-key mask.  One CTA per (history, head).  The forward
//                                                    streams keys through shared memory with an online softmax; the backward
//                                                    gives each warp every fourth key (dK, dV of that key summed over the T
//                                                    queries) and sums the warps' dQ partials in a fixed order.
// Dropout bits are te_keep of csrc/t5_dropout.cuh keyed on (history, head, query position, key position), the key position of a
// cross-attention key being its ORIGINAL encoder position, so both key layouts draw the same bits.  No global atomics: the
// gradients are bit-reproducible.
#include <cfloat>

#include "common.cuh"
#include "t5_dropout.cuh"

#define T5_DKV 64           // d_kv: every model EncoderDecoderRetrievalModel builds uses the T5Config default
#define T5_MAX_H 8          // positions of the self-attention cache (hierarchy levels)
#define XA_TILE 32          // encoder keys per shared-memory tile
#define XA_WARPS 4
#define XA_QPW 8            // queries per warp
#define XA_MAX_NQ (XA_WARPS * XA_QPW)

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------------ cross-attention
// grid (heads, B, ceil(nq / 32)), XA_WARPS warps: CTA z takes the history's queries 32 z .. 32 z + 31, so a query's arithmetic
// does not depend on nq.  q row b * nq + i, head n: q[(b * nq + i) * ldq + n * 64 + d]; key s of history b:
// k[(b * S + s) * ldkv + n * 64 + d] (v likewise); mask[b * S + s] == 0 masks the key (mask may be null); out like q.
__global__ void __launch_bounds__(XA_WARPS * 32) t5dec_cross_attention_kernel(
    const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, const float* __restrict__ v, int64_t ldkv,
    const float* __restrict__ mask, int nq, int S, float* __restrict__ out, int64_t ldo) {
  __shared__ float sq[XA_MAX_NQ][T5_DKV];
  __shared__ float sk[XA_TILE][T5_DKV + 1];   // +1: lane j reads row j, column d -> distinct banks
  __shared__ float sv[XA_TILE][T5_DKV];
  __shared__ float sbias[XA_TILE];
  const int n = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t col = (int64_t)n * T5_DKV;
  const int64_t row0 = (int64_t)b * nq + (int64_t)blockIdx.z * XA_MAX_NQ;     // this CTA's first query row
  const int ng = min(XA_MAX_NQ, nq - (int)blockIdx.z * XA_MAX_NQ);            // and its queries
  for (int i = threadIdx.x; i < ng * T5_DKV; i += blockDim.x)
    sq[i / T5_DKV][i % T5_DKV] = q[(row0 + i / T5_DKV) * ldq + col + i % T5_DKV];

  float m[XA_QPW], l[XA_QPW], acc0[XA_QPW], acc1[XA_QPW];
#pragma unroll
  for (int t = 0; t < XA_QPW; ++t) { m[t] = -INFINITY; l[t] = 0.f; acc0[t] = 0.f; acc1[t] = 0.f; }

  const float* kb = k + (int64_t)b * S * ldkv + col;
  const float* vb = v + (int64_t)b * S * ldkv + col;
  for (int s0 = 0; s0 < S; s0 += XA_TILE) {
    __syncthreads();                                        // the previous tile is consumed (and sq is written)
    for (int i = threadIdx.x; i < XA_TILE * T5_DKV; i += blockDim.x) {
      const int j = i / T5_DKV, d = i % T5_DKV, s = s0 + j;
      sk[j][d] = s < S ? kb[(int64_t)s * ldkv + d] : 0.f;
      sv[j][d] = s < S ? vb[(int64_t)s * ldkv + d] : 0.f;
    }
    if (threadIdx.x < XA_TILE) {
      const int s = s0 + threadIdx.x;
      sbias[threadIdx.x] = s >= S ? -INFINITY : (mask && mask[(int64_t)b * S + s] == 0.f ? -FLT_MAX : 0.f);
    }
    __syncthreads();
#pragma unroll
    for (int t = 0; t < XA_QPW; ++t) {
      const int qi = warp + t * XA_WARPS;
      if (qi >= ng) continue;
      float dot = 0.f;
#pragma unroll 16
      for (int d = 0; d < T5_DKV; ++d) dot = fmaf(sq[qi][d], sk[lane][d], dot);
      const float bias = sbias[lane];
      const float sc = bias == -INFINITY ? -INFINITY : dot + bias;   // a key past S contributes exp(-inf) = 0
      const float m_new = fmaxf(m[t], warp_max(sc));                // finite: every tile holds at least one key < S
      const float alpha = expf(m[t] - m_new);
      const float p = expf(sc - m_new);
      l[t] = l[t] * alpha + warp_sum(p);
      float a0 = acc0[t] * alpha, a1 = acc1[t] * alpha;
#pragma unroll 8
      for (int j = 0; j < XA_TILE; ++j) {
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
  for (int t = 0; t < XA_QPW; ++t) {
    const int qi = warp + t * XA_WARPS;
    if (qi >= ng) continue;
    float* o = out + (row0 + qi) * ldo + col;
    o[lane] = acc0[t] / l[t];
    o[lane + 32] = acc1[t] / l[t];
  }
}

// ------------------------------------------------------------------------------------------------ self-attention step
// One warp per (row r, head n); lane holds dims lane and lane + 32.  qkv row r: q at n * 64, k at inner + n * 64, v at
// 2 inner + n * 64.  cache slot j, row x, head n: cache[j * slot_stride + x * inner + n * 64 + d].  bias [heads, H, H]: the
// relative-position bias table of decoder block 0 (HF's compute_bias(H, H)), query position h.  LIVE: the grid is sized for R
// rows (the capacity) and the rows are the first min(*live, R); the warps of the others exit.
template <bool LIVE>
__global__ void __launch_bounds__(256) t5dec_self_attention_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, float* __restrict__ cache_k, float* __restrict__ cache_v, int64_t slot_stride,
    const float* __restrict__ bias, const int* __restrict__ anc_in, const int64_t* __restrict__ parent, int* __restrict__ anc_out,
    int R, int heads, int h, int H, float* __restrict__ out, int64_t ldo, const int* __restrict__ live) {
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (LIVE) R = min(R, max(0, *live));
  if (gw >= R * heads) return;
  const int r = gw / heads, n = gw % heads;
  const int inner = heads * T5_DKV;
  const float* row = qkv + (int64_t)r * ldqkv + n * T5_DKV;
  const float q0 = row[lane], q1 = row[lane + 32];
  const float k0 = row[inner + lane], k1 = row[inner + lane + 32];
  const float v0 = row[2 * inner + lane], v1 = row[2 * inner + lane + 32];
  const int64_t here = (int64_t)h * slot_stride + (int64_t)r * inner + n * T5_DKV;
  cache_k[here + lane] = k0;
  cache_k[here + lane + 32] = k1;
  cache_v[here + lane] = v0;
  cache_v[here + lane + 32] = v1;

  // ancestors: lane j < h holds the row of slot j this beam reads
  int anc = 0;
  if (lane < h) {
    if (parent) {
      const int64_t p = parent[r];
      anc = lane == h - 1 ? (int)p : anc_in[p * H + lane];
      if (n == 0) anc_out[(int64_t)r * H + lane] = anc;
    } else {
      anc = anc_in[(int64_t)r * H + lane];
    }
  }
  const float* brow = bias + ((int64_t)n * H + h) * H;
  float sc[T5_MAX_H];
  float mx = warp_sum(fmaf(q0, k0, q1 * k1)) + brow[h];
  sc[0] = mx;                                               // sc[0] is position h, sc[1 + j] position j
#pragma unroll
  for (int j = 0; j < T5_MAX_H - 1; ++j) {
    if (j >= h) break;
    const int x = __shfl_sync(0xffffffffu, anc, j);
    const float* kj = cache_k + (int64_t)j * slot_stride + (int64_t)x * inner + n * T5_DKV;
    sc[1 + j] = warp_sum(fmaf(q0, kj[lane], q1 * kj[lane + 32])) + brow[j];
    mx = fmaxf(mx, sc[1 + j]);
  }
  float p = expf(sc[0] - mx);
  float sum = p, o0 = p * v0, o1 = p * v1;
#pragma unroll
  for (int j = 0; j < T5_MAX_H - 1; ++j) {
    if (j >= h) break;
    const int x = __shfl_sync(0xffffffffu, anc, j);
    const float* vj = cache_v + (int64_t)j * slot_stride + (int64_t)x * inner + n * T5_DKV;
    p = expf(sc[1 + j] - mx);
    sum += p;
    o0 = fmaf(p, vj[lane], o0);
    o1 = fmaf(p, vj[lane + 32], o1);
  }
  float* o = out + (int64_t)r * ldo + n * T5_DKV;
  o[lane] = o0 / sum;
  o[lane + 32] = o1 / sum;
}

// ------------------------------------------------------------------------------------------------ residual add + T5LayerNorm
// One warp per row.  emb != null: x[r] = emb[(ids ? ids[r * ids_stride] + id_offset : 0)] (an id outside [0, n_emb) gives a NaN
// row); else delta != null: x[r] += delta[r].  Then out[r] = weight * (x * rsqrt(mean(x^2) + eps)).  LIVE as the self-attention.
template <bool LIVE>
__global__ void __launch_bounds__(256) t5dec_add_norm_kernel(
    float* __restrict__ x, const float* __restrict__ delta, int64_t ld_delta, const float* __restrict__ emb,
    const int64_t* __restrict__ ids, int64_t ids_stride, int64_t id_offset, int64_t n_emb, const float* __restrict__ weight,
    int R, int D, float eps, float* __restrict__ out, const int* __restrict__ live) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (LIVE) R = min(R, max(0, *live));
  if (r >= R) return;
  float* xr = x + (int64_t)r * D;
  float ss = 0.f;
  if (emb) {
    const int64_t id = ids ? ids[(int64_t)r * ids_stride] + id_offset : 0;
    const bool ok = id >= 0 && id < n_emb;
    const float* er = emb + (ok ? id : 0) * D;
    for (int d = lane; d < D; d += 32) {
      const float val = ok ? er[d] : __int_as_float(0x7fffffff);
      xr[d] = val;
      ss = fmaf(val, val, ss);
    }
  } else {
    const float* dr = delta ? delta + (int64_t)r * ld_delta : nullptr;
    for (int d = lane; d < D; d += 32) {
      const float val = dr ? xr[d] + dr[d] : xr[d];
      xr[d] = val;
      ss = fmaf(val, val, ss);
    }
  }
  const float inv = rsqrtf(warp_sum(ss) / (float)D + eps);
  __syncwarp();
  float* orow = out + (int64_t)r * D;
  for (int d = lane; d < D; d += 32) orow[d] = weight[d] * (xr[d] * inv);
}

// ------------------------------------------------------------------------------------------------ training: causal self-attention
// One warp per (history b, head n); lane holds dims lane and lane + 32 of each of the history's T rows.  qkv row b * T + t: q at
// n * 64, k at inner + n * 64, v at 2 inner + n * 64.  rel [heads, 2T - 1]: the bias of key j for query t is rel[n, j - t + T - 1].
// Keys after the query are skipped (HF gives them weight exactly 0).  out like q; lse[(b * T + t) * heads + n] = m + log l.
__global__ void __launch_bounds__(256) t5dec_self_attention_train_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, const float* __restrict__ rel, int B, int T, int heads,
    const int64_t* __restrict__ seed, uint32_t thresh, float scale, float* __restrict__ out, int64_t ldo, float* __restrict__ lse) {
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (gw >= B * heads) return;
  const int b = gw / heads, n = gw % heads;
  const int64_t inner = (int64_t)heads * T5_DKV;
  const float* relr = rel + (int64_t)n * (2 * T - 1) + (T - 1);   // relr[j - t]
  const uint2 key = thresh ? te_seed_key(seed) : make_uint2(0u, 0u);
  float k0[T5_MAX_H], k1[T5_MAX_H], v0[T5_MAX_H], v1[T5_MAX_H];
#pragma unroll
  for (int j = 0; j < T5_MAX_H; ++j) {
    k0[j] = k1[j] = v0[j] = v1[j] = 0.f;
    if (j < T) {
      const float* row = qkv + ((int64_t)b * T + j) * ldqkv + n * T5_DKV;
      k0[j] = row[inner + lane];
      k1[j] = row[inner + lane + 32];
      v0[j] = row[2 * inner + lane];
      v1[j] = row[2 * inner + lane + 32];
    }
  }
  for (int t = 0; t < T; ++t) {
    const int64_t r = (int64_t)b * T + t;
    const float q0 = qkv[r * ldqkv + n * T5_DKV + lane], q1 = qkv[r * ldqkv + n * T5_DKV + lane + 32];
    float s[T5_MAX_H];
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < T5_MAX_H; ++j) {
      s[j] = -INFINITY;
      if (j <= t) {
        s[j] = warp_sum(fmaf(q0, k0[j], q1 * k1[j])) + relr[j - t];
        m = fmaxf(m, s[j]);
      }
    }
    float l = 0.f, o0 = 0.f, o1 = 0.f;
#pragma unroll
    for (int j = 0; j < T5_MAX_H; ++j) {
      if (j <= t) {
        float p = expf(s[j] - m);
        l += p;
        if (thresh && !te_keep(key, b, n, t, j, thresh)) p = 0.f;
        o0 = fmaf(p, v0[j], o0);
        o1 = fmaf(p, v1[j], o1);
      }
    }
    float* orow = out + r * ldo + n * T5_DKV;
    orow[lane] = thresh ? o0 / l * scale : o0 / l;
    orow[lane + 32] = thresh ? o1 / l * scale : o1 / l;
    if (lane == 0) lse[r * heads + n] = m + logf(l);
  }
}

// The backward, same layout: dS_tj = P_tj (dP_tj z_tj - D_t) with z the kept weights' scale (0 when dropped), dP_tj = dO_t . v_j,
// D_t = dO_t . O_t and P_tj = exp(s_tj - lse_t).  Writes dQ | dK | dV into dqkv and drel_part[(b * heads + n) * (2T - 1) + i], the
// warp's sum of dS at distance i - (T - 1) (0 for the positive distances causality never reaches), summed in (t, j) order.
__global__ void __launch_bounds__(256) t5dec_self_attention_bwd_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, const float* __restrict__ o, int64_t ldo, const float* __restrict__ dout,
    int64_t lddo, const float* __restrict__ lse, const float* __restrict__ rel, int B, int T, int heads,
    const int64_t* __restrict__ seed, uint32_t thresh, float scale, float* __restrict__ dqkv, int64_t ldd,
    float* __restrict__ drel_part) {
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (gw >= B * heads) return;
  const int b = gw / heads, n = gw % heads;
  const int64_t inner = (int64_t)heads * T5_DKV;
  const float* relr = rel + (int64_t)n * (2 * T - 1) + (T - 1);
  const uint2 key = thresh ? te_seed_key(seed) : make_uint2(0u, 0u);
  float k0[T5_MAX_H], k1[T5_MAX_H], v0[T5_MAX_H], v1[T5_MAX_H];
  float dk0[T5_MAX_H], dk1[T5_MAX_H], dv0[T5_MAX_H], dv1[T5_MAX_H];
#pragma unroll
  for (int j = 0; j < T5_MAX_H; ++j) {
    k0[j] = k1[j] = v0[j] = v1[j] = 0.f;
    dk0[j] = dk1[j] = dv0[j] = dv1[j] = 0.f;
    if (j < T) {
      const float* row = qkv + ((int64_t)b * T + j) * ldqkv + n * T5_DKV;
      k0[j] = row[inner + lane];
      k1[j] = row[inner + lane + 32];
      v0[j] = row[2 * inner + lane];
      v1[j] = row[2 * inner + lane + 32];
    }
  }
  float bin = 0.f;                                          // lane i < T: the sum of dS at distance t - j = i
  for (int t = 0; t < T; ++t) {
    const int64_t r = (int64_t)b * T + t;
    const float q0 = qkv[r * ldqkv + n * T5_DKV + lane], q1 = qkv[r * ldqkv + n * T5_DKV + lane + 32];
    const float g0 = dout[r * lddo + n * T5_DKV + lane], g1 = dout[r * lddo + n * T5_DKV + lane + 32];
    const float di = warp_sum(fmaf(g0, o[r * ldo + n * T5_DKV + lane], g1 * o[r * ldo + n * T5_DKV + lane + 32]));
    const float li = lse[r * heads + n];
    float dq0 = 0.f, dq1 = 0.f;
#pragma unroll
    for (int j = 0; j < T5_MAX_H; ++j) {
      if (j <= t) {
        const float s = warp_sum(fmaf(q0, k0[j], q1 * k1[j])) + relr[j - t];
        const float p = expf(s - li);
        const float z = thresh ? (te_keep(key, b, n, t, j, thresh) ? scale : 0.f) : 1.f;
        const float ds = p * (warp_sum(fmaf(g0, v0[j], g1 * v1[j])) * z - di);
        dq0 = fmaf(ds, k0[j], dq0);
        dq1 = fmaf(ds, k1[j], dq1);
        dk0[j] = fmaf(ds, q0, dk0[j]);
        dk1[j] = fmaf(ds, q1, dk1[j]);
        dv0[j] = fmaf(p * z, g0, dv0[j]);
        dv1[j] = fmaf(p * z, g1, dv1[j]);
        if (lane == t - j) bin += ds;
      }
    }
    dqkv[r * ldd + n * T5_DKV + lane] = dq0;
    dqkv[r * ldd + n * T5_DKV + lane + 32] = dq1;
  }
#pragma unroll
  for (int j = 0; j < T5_MAX_H; ++j) {
    if (j < T) {
      float* row = dqkv + ((int64_t)b * T + j) * ldd + n * T5_DKV;
      row[inner + lane] = dk0[j];
      row[inner + lane + 32] = dk1[j];
      row[2 * inner + lane] = dv0[j];
      row[2 * inner + lane + 32] = dv1[j];
    }
  }
  const float mine = __shfl_sync(0xffffffffu, bin, (T - 1 - lane) & 31);   // entry i = lane holds distance i - (T - 1)
  if (lane < 2 * T - 1) drel_part[((int64_t)b * heads + n) * (2 * T - 1) + lane] = lane < T ? mine : 0.f;
}

// ------------------------------------------------------------------------------------------------ training: cross-attention
// grid (B, heads), XA_WARPS warps.  q row b * T + t; key rows offsets[b] .. offsets[b + 1] - 1 of k / v (row stride ldkv) with the
// additive mask key_mask[row] (0 or -FLT_MAX) and original position src[row] - b * S (src null: row - offsets[b]).  The score is
// q . k + key_mask; lse[(b * T + t) * heads + n] = (m - base) + log l with base the largest key_mask of the history, so a history
// whose keys are all masked keeps a finite lse that the backward's exp((s - base) - lse) turns back into its uniform weights.
#define XT_QPW ((T5_MAX_H + XA_WARPS - 1) / XA_WARPS)      // decoder queries per warp

__device__ __forceinline__ int xt_pos(const int* src, int row, int b, int S, int off) {
  return src ? src[row] - b * S : row - off;
}

__global__ void __launch_bounds__(XA_WARPS * 32) t5dec_cross_attention_train_kernel(
    const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, const float* __restrict__ v, int64_t ldkv,
    const int* __restrict__ offsets, const float* __restrict__ key_mask, const int* __restrict__ src, int S, int T, int heads,
    const int64_t* __restrict__ seed, uint32_t thresh, float scale, float* __restrict__ out, int64_t ldo, float* __restrict__ lse) {
  __shared__ float sq[T5_MAX_H][T5_DKV];
  __shared__ float sk[XA_TILE][T5_DKV + 1];
  __shared__ float sv[XA_TILE][T5_DKV];
  __shared__ float smask[XA_TILE];
  __shared__ int spos[XA_TILE];
  const int b = blockIdx.x, n = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t col = (int64_t)n * T5_DKV;
  const int off = offsets[b], cnt = offsets[b + 1] - off;
  for (int i = threadIdx.x; i < T * T5_DKV; i += blockDim.x)
    sq[i / T5_DKV][i % T5_DKV] = q[((int64_t)b * T + i / T5_DKV) * ldq + col + i % T5_DKV];
  const uint2 key = thresh ? te_seed_key(seed) : make_uint2(0u, 0u);

  float m[XT_QPW], l[XT_QPW], acc0[XT_QPW], acc1[XT_QPW];
#pragma unroll
  for (int u = 0; u < XT_QPW; ++u) { m[u] = -INFINITY; l[u] = 0.f; acc0[u] = 0.f; acc1[u] = 0.f; }
  float base = -INFINITY;
  for (int s0 = 0; s0 < cnt; s0 += XA_TILE) {
    __syncthreads();                                        // the previous tile is consumed (and sq is written)
    for (int i = threadIdx.x; i < XA_TILE * T5_DKV; i += blockDim.x) {
      const int j = i / T5_DKV, d = i % T5_DKV, s = s0 + j;
      sk[j][d] = s < cnt ? k[(int64_t)(off + s) * ldkv + col + d] : 0.f;
      sv[j][d] = s < cnt ? v[(int64_t)(off + s) * ldkv + col + d] : 0.f;
    }
    if (threadIdx.x < XA_TILE) {
      const int s = s0 + threadIdx.x;
      smask[threadIdx.x] = s < cnt ? key_mask[off + s] : -INFINITY;
      spos[threadIdx.x] = s < cnt ? xt_pos(src, off + s, b, S, off) : 0;
    }
    __syncthreads();
    const float mk = smask[lane];
    const int pos = spos[lane];
    base = fmaxf(base, warp_max(mk));
#pragma unroll
    for (int u = 0; u < XT_QPW; ++u) {
      const int t = warp + u * XA_WARPS;
      if (t >= T) continue;
      float dot = 0.f;
#pragma unroll 16
      for (int d = 0; d < T5_DKV; ++d) dot = fmaf(sq[t][d], sk[lane][d], dot);
      const float sc = mk == -INFINITY ? -INFINITY : dot + mk;     // a key past the history contributes exp(-inf) = 0
      const float m_new = fmaxf(m[u], warp_max(sc));              // finite: every tile holds at least one key of the history
      const float alpha = expf(m[u] - m_new);
      float p = expf(sc - m_new);
      l[u] = l[u] * alpha + warp_sum(p);
      if (thresh && mk != -INFINITY && !te_keep(key, b, n, t, pos, thresh)) p = 0.f;
      float a0 = acc0[u] * alpha, a1 = acc1[u] * alpha;
#pragma unroll 8
      for (int j = 0; j < XA_TILE; ++j) {
        const float pj = __shfl_sync(0xffffffffu, p, j);
        a0 = fmaf(pj, sv[j][lane], a0);
        a1 = fmaf(pj, sv[j][lane + 32], a1);
      }
      acc0[u] = a0;
      acc1[u] = a1;
      m[u] = m_new;
    }
  }
#pragma unroll
  for (int u = 0; u < XT_QPW; ++u) {
    const int t = warp + u * XA_WARPS;
    if (t >= T) continue;
    const int64_t r = (int64_t)b * T + t;
    float* orow = out + r * ldo + col;
    if (cnt == 0) {                                         // a history without keys: zeros
      orow[lane] = orow[lane + 32] = 0.f;
      if (lane == 0) lse[r * heads + n] = 0.f;
      continue;
    }
    orow[lane] = thresh ? acc0[u] / l[u] * scale : acc0[u] / l[u];
    orow[lane + 32] = thresh ? acc1[u] / l[u] * scale : acc1[u] / l[u];
    if (lane == 0) lse[r * heads + n] = (m[u] - base) + logf(l[u]);
  }
}

// grid (B, heads), XA_WARPS warps.  Warp w takes keys w, w + XA_WARPS, ... of the history in order, lane holding dims lane and
// lane + 32: dK / dV of the key are its sums over the T queries, written directly; dQ partials stay per warp and are summed over
// the warps in order at the end.  dS_tk = P_tk (dP_tk z_tk - D_t), P_tk = exp((s_tk - base) - lse_t), D_t = dO_t . O_t.
__global__ void __launch_bounds__(XA_WARPS * 32) t5dec_cross_attention_bwd_kernel(
    const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, const float* __restrict__ v, int64_t ldkv,
    const float* __restrict__ o, int64_t ldo, const float* __restrict__ dout, int64_t lddo, const float* __restrict__ lse,
    const int* __restrict__ offsets, const float* __restrict__ key_mask, const int* __restrict__ src, int S, int T, int heads,
    const int64_t* __restrict__ seed, uint32_t thresh, float scale, float* __restrict__ dq, int64_t lddq, float* __restrict__ dk,
    float* __restrict__ dv, int64_t lddkv) {
  __shared__ float sdq[XA_WARPS][T5_MAX_H][T5_DKV];
  __shared__ float sdi[T5_MAX_H], slse[T5_MAX_H];
  __shared__ float sbase[XA_WARPS];
  const int b = blockIdx.x, n = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t col = (int64_t)n * T5_DKV;
  const int off = offsets[b], cnt = offsets[b + 1] - off;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < cnt; i += blockDim.x) mx = fmaxf(mx, key_mask[off + i]);
  mx = warp_max(mx);
  if (lane == 0) sbase[warp] = mx;
  for (int t = warp; t < T; t += XA_WARPS) {
    const int64_t r = (int64_t)b * T + t;
    const float di = warp_sum(fmaf(dout[r * lddo + col + lane], o[r * ldo + col + lane],
                                   dout[r * lddo + col + lane + 32] * o[r * ldo + col + lane + 32]));
    if (lane == 0) {
      sdi[t] = di;
      slse[t] = lse[r * heads + n];
    }
  }
  __syncthreads();
  float base = sbase[0];
#pragma unroll
  for (int w = 1; w < XA_WARPS; ++w) base = fmaxf(base, sbase[w]);
  const uint2 key = thresh ? te_seed_key(seed) : make_uint2(0u, 0u);

  float q0[T5_MAX_H], q1[T5_MAX_H], g0[T5_MAX_H], g1[T5_MAX_H], dq0[T5_MAX_H], dq1[T5_MAX_H];
#pragma unroll
  for (int t = 0; t < T5_MAX_H; ++t) {
    q0[t] = q1[t] = g0[t] = g1[t] = dq0[t] = dq1[t] = 0.f;
    if (t < T) {
      const int64_t r = (int64_t)b * T + t;
      q0[t] = q[r * ldq + col + lane];
      q1[t] = q[r * ldq + col + lane + 32];
      g0[t] = dout[r * lddo + col + lane];
      g1[t] = dout[r * lddo + col + lane + 32];
    }
  }
  for (int s = warp; s < cnt; s += XA_WARPS) {
    const int64_t row = off + s;
    const float k0 = k[row * ldkv + col + lane], k1 = k[row * ldkv + col + lane + 32];
    const float v0 = v[row * ldkv + col + lane], v1 = v[row * ldkv + col + lane + 32];
    const float mk = key_mask[row];
    const int pos = xt_pos(src, (int)row, b, S, off);
    float dk0 = 0.f, dk1 = 0.f, dv0 = 0.f, dv1 = 0.f;
#pragma unroll
    for (int t = 0; t < T5_MAX_H; ++t) {
      if (t < T) {
        const float sc = warp_sum(fmaf(q0[t], k0, q1[t] * k1)) + mk;
        const float p = expf((sc - base) - slse[t]);
        const float z = thresh ? (te_keep(key, b, n, t, pos, thresh) ? scale : 0.f) : 1.f;
        const float ds = p * (warp_sum(fmaf(g0[t], v0, g1[t] * v1)) * z - sdi[t]);
        dq0[t] = fmaf(ds, k0, dq0[t]);
        dq1[t] = fmaf(ds, k1, dq1[t]);
        dk0 = fmaf(ds, q0[t], dk0);
        dk1 = fmaf(ds, q1[t], dk1);
        dv0 = fmaf(p * z, g0[t], dv0);
        dv1 = fmaf(p * z, g1[t], dv1);
      }
    }
    dk[row * lddkv + col + lane] = dk0;
    dk[row * lddkv + col + lane + 32] = dk1;
    dv[row * lddkv + col + lane] = dv0;
    dv[row * lddkv + col + lane + 32] = dv1;
  }
#pragma unroll
  for (int t = 0; t < T5_MAX_H; ++t) {
    if (t < T) {
      sdq[warp][t][lane] = dq0[t];
      sdq[warp][t][lane + 32] = dq1[t];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < T * T5_DKV; i += blockDim.x) {
    const int t = i / T5_DKV, d = i % T5_DKV;
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < XA_WARPS; ++w) acc += sdq[w][t][d];
    dq[((int64_t)b * T + t) * lddq + col + d] = acc;
  }
}

// ------------------------------------------------------------------------------------------------ C ABI
extern "C" int rqb200_t5dec_cross_attention(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv,
                                            const float* mask, int B, int nq, int S, int heads, float* out, int64_t ldo,
                                            void* stream) {
  RQB_CHECK_ARG(B >= 0 && nq > 0 && S > 0 && heads > 0, "t5dec_cross_attention: bad shape (B=%d nq=%d S=%d heads=%d)", B, nq,
                S, heads);
  const int groups = (nq + XA_MAX_NQ - 1) / XA_MAX_NQ;
  if (groups > 65535 || B > 65535) {
    rqb_set_error("t5dec_cross_attention: need nq <= %d queries per history and B <= 65535 (nq = %d, B = %d)", 65535 * XA_MAX_NQ,
                  nq, B);
    return RQB_ERR_UNSUPPORTED;
  }
  const int64_t inner = (int64_t)heads * T5_DKV;
  RQB_CHECK_ARG(ldq >= inner && ldkv >= inner && ldo >= inner, "t5dec_cross_attention: a leading dimension is below heads * 64");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(q && k && v && out, "t5dec_cross_attention: null pointer");
  t5dec_cross_attention_kernel<<<dim3(heads, B, groups), XA_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      q, ldq, k, v, ldkv, mask, nq, S, out, ldo);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

template <bool LIVE>
static int dec_self_attention(const char* what, const float* qkv, int64_t ldqkv, float* cache_k, float* cache_v, int64_t slot_stride,
                              const float* bias, const int* anc_in, const int64_t* parent, int* anc_out, int R, int heads, int h,
                              int H, float* out, int64_t ldo, const int* live, void* stream) {
  RQB_CHECK_ARG(R >= 0 && heads > 0 && h >= 0 && h < H, "%s: bad shape (R=%d heads=%d h=%d H=%d)", what, R, heads, h, H);
  if (H > T5_MAX_H) {
    rqb_set_error("%s: at most %d positions (H = %d)", what, T5_MAX_H, H);
    return RQB_ERR_UNSUPPORTED;
  }
  const int64_t inner = (int64_t)heads * T5_DKV;
  RQB_CHECK_ARG(ldqkv >= 3 * inner && ldo >= inner && slot_stride >= (int64_t)R * inner,
                "%s: a leading dimension or the slot stride is too small", what);
  if (R == 0) return RQB_OK;
  RQB_CHECK_ARG(qkv && cache_k && cache_v && bias && out && (live || !LIVE), "%s: null pointer", what);
  RQB_CHECK_ARG(h == 0 || (anc_in && (!parent || anc_out)), "%s: h > 0 needs the ancestor table", what);
  const int64_t warps = (int64_t)R * heads;
  RQB_CHECK_ARG(warps <= (int64_t)INT32_MAX - 7, "%s: too many rows", what);
  t5dec_self_attention_kernel<LIVE><<<(unsigned)((warps + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      qkv, ldqkv, cache_k, cache_v, slot_stride, bias, anc_in, parent, anc_out, R, heads, h, H, out, ldo, live);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5dec_self_attention(const float* qkv, int64_t ldqkv, float* cache_k, float* cache_v, int64_t slot_stride,
                                           const float* bias, const int* anc_in, const int64_t* parent, int* anc_out, int R,
                                           int heads, int h, int H, float* out, int64_t ldo, void* stream) {
  return dec_self_attention<false>("t5dec_self_attention", qkv, ldqkv, cache_k, cache_v, slot_stride, bias, anc_in, parent, anc_out,
                                   R, heads, h, H, out, ldo, nullptr, stream);
}

extern "C" int rqb200_t5dec_self_attention_counted(const float* qkv, int64_t ldqkv, float* cache_k, float* cache_v,
                                                   int64_t slot_stride, const float* bias, const int* anc_in, const int64_t* parent,
                                                   int* anc_out, int R, const int* live_r, int heads, int h, int H, float* out,
                                                   int64_t ldo, void* stream) {
  return dec_self_attention<true>("t5dec_self_attention_counted", qkv, ldqkv, cache_k, cache_v, slot_stride, bias, anc_in, parent,
                                  anc_out, R, heads, h, H, out, ldo, live_r, stream);
}

template <bool LIVE>
static int dec_add_norm(const char* what, float* x, const float* delta, int64_t ld_delta, const float* emb, const int64_t* ids,
                        int64_t ids_stride, int64_t id_offset, int64_t n_emb, const float* weight, int R, int D, float eps, float* out,
                        const int* live, void* stream) {
  RQB_CHECK_ARG(R >= 0 && D > 0 && (!delta || ld_delta >= D) && (!emb || n_emb > 0), "%s: bad shape (R=%d D=%d)", what, R, D);
  if (R == 0) return RQB_OK;
  RQB_CHECK_ARG(x && weight && out && (live || !LIVE), "%s: null pointer", what);
  t5dec_add_norm_kernel<LIVE><<<(R + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, delta, ld_delta, emb, ids, ids_stride, id_offset, n_emb, weight, R, D, eps, out, live);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5dec_add_norm(float* x, const float* delta, int64_t ld_delta, const float* emb, const int64_t* ids,
                                     int64_t ids_stride, int64_t id_offset, int64_t n_emb, const float* weight, int R, int D,
                                     float eps, float* out, void* stream) {
  return dec_add_norm<false>("t5dec_add_norm", x, delta, ld_delta, emb, ids, ids_stride, id_offset, n_emb, weight, R, D, eps, out,
                             nullptr, stream);
}

extern "C" int rqb200_t5dec_add_norm_counted(float* x, const float* delta, int64_t ld_delta, const float* emb, const int64_t* ids,
                                             int64_t ids_stride, int64_t id_offset, int64_t n_emb, const float* weight, int R,
                                             const int* live_r, int D, float eps, float* out, void* stream) {
  return dec_add_norm<true>("t5dec_add_norm_counted", x, delta, ld_delta, emb, ids, ids_stride, id_offset, n_emb, weight, R, D, eps,
                            out, live_r, stream);
}

static int dec_train_args(int B, int T, int heads, float p, const char* what) {
  RQB_CHECK_ARG(B >= 0 && T > 0 && heads > 0, "%s: bad shape (B=%d T=%d heads=%d)", what, B, T, heads);
  RQB_CHECK_ARG(p >= 0.f && p < 1.f, "%s: dropout probability %g outside [0, 1)", what, (double)p);
  if (T > T5_MAX_H) {
    rqb_set_error("%s: at most %d decoder positions (T = %d)", what, T5_MAX_H, T);
    return RQB_ERR_UNSUPPORTED;
  }
  RQB_CHECK_ARG(B <= INT32_MAX / T && (int64_t)B * heads <= (int64_t)INT32_MAX - 7, "%s: too many histories", what);
  return RQB_OK;
}

extern "C" int rqb200_t5dec_self_attention_train(const float* qkv, int64_t ldqkv, const float* rel, int B, int T, int heads,
                                                 const int64_t* seed, float p, float* out, int64_t ldo, float* lse, void* stream) {
  if (int rc = dec_train_args(B, T, heads, p, "t5dec_self_attention_train")) return rc;
  const int64_t inner = (int64_t)heads * T5_DKV;
  RQB_CHECK_ARG(ldqkv >= 3 * inner && ldo >= inner, "t5dec_self_attention_train: a leading dimension is too small");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(qkv && rel && seed && out && lse, "t5dec_self_attention_train: null pointer");
  uint32_t thresh;
  float scale;
  dropout_params(p, &thresh, &scale);
  const int64_t warps = (int64_t)B * heads;
  t5dec_self_attention_train_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      qkv, ldqkv, rel, B, T, heads, seed, thresh, scale, out, ldo, lse);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5dec_self_attention_backward(const float* qkv, int64_t ldqkv, const float* out, int64_t ldo,
                                                    const float* dout, int64_t lddo, const float* lse, const float* rel, int B, int T,
                                                    int heads, const int64_t* seed, float p, float* dqkv, int64_t ldd,
                                                    float* drel_part, void* stream) {
  if (int rc = dec_train_args(B, T, heads, p, "t5dec_self_attention_backward")) return rc;
  const int64_t inner = (int64_t)heads * T5_DKV;
  RQB_CHECK_ARG(ldqkv >= 3 * inner && ldo >= inner && lddo >= inner && ldd >= 3 * inner,
                "t5dec_self_attention_backward: a leading dimension is too small");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(qkv && out && dout && lse && rel && seed && dqkv && drel_part, "t5dec_self_attention_backward: null pointer");
  uint32_t thresh;
  float scale;
  dropout_params(p, &thresh, &scale);
  const int64_t warps = (int64_t)B * heads;
  t5dec_self_attention_bwd_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      qkv, ldqkv, out, ldo, dout, lddo, lse, rel, B, T, heads, seed, thresh, scale, dqkv, ldd, drel_part);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

static int cross_train_args(int B, int S, int T, int heads, float p, const char* what) {
  if (int rc = dec_train_args(B, T, heads, p, what)) return rc;
  RQB_CHECK_ARG(S > 0 && heads <= 65535, "%s: bad shape (S=%d heads=%d)", what, S, heads);
  return RQB_OK;
}

extern "C" int rqb200_t5dec_cross_attention_train(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv,
                                                  const int* offsets, const float* key_mask, const int* src, int B, int S, int T,
                                                  int heads, const int64_t* seed, float p, float* out, int64_t ldo, float* lse,
                                                  void* stream) {
  if (int rc = cross_train_args(B, S, T, heads, p, "t5dec_cross_attention_train")) return rc;
  const int64_t inner = (int64_t)heads * T5_DKV;
  RQB_CHECK_ARG(ldq >= inner && ldkv >= inner && ldo >= inner, "t5dec_cross_attention_train: a leading dimension is below heads * 64");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(q && k && v && offsets && key_mask && seed && out && lse, "t5dec_cross_attention_train: null pointer");
  uint32_t thresh;
  float scale;
  dropout_params(p, &thresh, &scale);
  t5dec_cross_attention_train_kernel<<<dim3(B, heads), XA_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      q, ldq, k, v, ldkv, offsets, key_mask, src, S, T, heads, seed, thresh, scale, out, ldo, lse);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5dec_cross_attention_backward(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv,
                                                     const float* out, int64_t ldo, const float* dout, int64_t lddo, const float* lse,
                                                     const int* offsets, const float* key_mask, const int* src, int B, int S, int T,
                                                     int heads, const int64_t* seed, float p, float* dq, int64_t lddq, float* dk,
                                                     float* dv, int64_t lddkv, void* stream) {
  if (int rc = cross_train_args(B, S, T, heads, p, "t5dec_cross_attention_backward")) return rc;
  const int64_t inner = (int64_t)heads * T5_DKV;
  RQB_CHECK_ARG(ldq >= inner && ldkv >= inner && ldo >= inner && lddo >= inner && lddq >= inner && lddkv >= inner,
                "t5dec_cross_attention_backward: a leading dimension is below heads * 64");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(q && k && v && out && dout && lse && offsets && key_mask && seed && dq && dk && dv,
                "t5dec_cross_attention_backward: null pointer");
  uint32_t thresh;
  float scale;
  dropout_params(p, &thresh, &scale);
  t5dec_cross_attention_bwd_kernel<<<dim3(B, heads), XA_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      q, ldq, k, v, ldkv, out, ldo, dout, lddo, lse, offsets, key_mask, src, S, T, heads, seed, thresh, scale, dq, lddq, dk, dv,
      lddkv);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}
