// One decoder step of the generative-retrieval model's T5 stack (transformers T5Stack in eval mode, is_decoder=True) for the
// fused decode path of EncoderDecoderRetrievalModel.generate(decoder="fused").  The GEMMs stay with cuBLAS; these kernels do
// what lies between them, without copying any key/value state:
//
//   rqb200_t5dec_cross_attention  attention over the encoder output, one CTA per (history, head).  Every beam of a history has the
//                                 same cross keys and values, so they are stored once per history ([B, S] rows) and the CTA reads
//                                 them once for all of the history's nq queries (1 at level 0, top_k later).  Keys stream through
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
#include <cfloat>

#include "common.cuh"

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
// grid (heads, B), XA_WARPS warps.  q row b * nq + i, head n: q[(b * nq + i) * ldq + n * 64 + d]; key s of history b:
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
  for (int i = threadIdx.x; i < nq * T5_DKV; i += blockDim.x)
    sq[i / T5_DKV][i % T5_DKV] = q[((int64_t)b * nq + i / T5_DKV) * ldq + col + i % T5_DKV];

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
      if (qi >= nq) continue;
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
    if (qi >= nq) continue;
    float* o = out + ((int64_t)b * nq + qi) * ldo + col;
    o[lane] = acc0[t] / l[t];
    o[lane + 32] = acc1[t] / l[t];
  }
}

// ------------------------------------------------------------------------------------------------ self-attention step
// One warp per (row r, head n); lane holds dims lane and lane + 32.  qkv row r: q at n * 64, k at inner + n * 64, v at
// 2 inner + n * 64.  cache slot j, row x, head n: cache[j * slot_stride + x * inner + n * 64 + d].  bias [heads, H, H]: the
// relative-position bias table of decoder block 0 (HF's compute_bias(H, H)), query position h.
__global__ void __launch_bounds__(256) t5dec_self_attention_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, float* __restrict__ cache_k, float* __restrict__ cache_v, int64_t slot_stride,
    const float* __restrict__ bias, const int* __restrict__ anc_in, const int64_t* __restrict__ parent, int* __restrict__ anc_out,
    int R, int heads, int h, int H, float* __restrict__ out, int64_t ldo) {
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
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
// row); else delta != null: x[r] += delta[r].  Then out[r] = weight * (x * rsqrt(mean(x^2) + eps)).
__global__ void __launch_bounds__(256) t5dec_add_norm_kernel(
    float* __restrict__ x, const float* __restrict__ delta, int64_t ld_delta, const float* __restrict__ emb,
    const int64_t* __restrict__ ids, int64_t ids_stride, int64_t id_offset, int64_t n_emb, const float* __restrict__ weight,
    int R, int D, float eps, float* __restrict__ out) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
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

// ------------------------------------------------------------------------------------------------ C ABI
extern "C" int rqb200_t5dec_cross_attention(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv,
                                            const float* mask, int B, int nq, int S, int heads, float* out, int64_t ldo,
                                            void* stream) {
  RQB_CHECK_ARG(B >= 0 && nq > 0 && S > 0 && heads > 0, "t5dec_cross_attention: bad shape (B=%d nq=%d S=%d heads=%d)", B, nq,
                S, heads);
  if (nq > XA_MAX_NQ || B > 65535) {
    rqb_set_error("t5dec_cross_attention: need nq <= %d queries per history and B <= 65535 (nq = %d, B = %d)", XA_MAX_NQ, nq, B);
    return RQB_ERR_UNSUPPORTED;
  }
  const int64_t inner = (int64_t)heads * T5_DKV;
  RQB_CHECK_ARG(ldq >= inner && ldkv >= inner && ldo >= inner, "t5dec_cross_attention: a leading dimension is below heads * 64");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(q && k && v && out, "t5dec_cross_attention: null pointer");
  t5dec_cross_attention_kernel<<<dim3(heads, B), XA_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      q, ldq, k, v, ldkv, mask, nq, S, out, ldo);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5dec_self_attention(const float* qkv, int64_t ldqkv, float* cache_k, float* cache_v, int64_t slot_stride,
                                           const float* bias, const int* anc_in, const int64_t* parent, int* anc_out, int R,
                                           int heads, int h, int H, float* out, int64_t ldo, void* stream) {
  RQB_CHECK_ARG(R >= 0 && heads > 0 && h >= 0 && h < H, "t5dec_self_attention: bad shape (R=%d heads=%d h=%d H=%d)", R, heads,
                h, H);
  if (H > T5_MAX_H) {
    rqb_set_error("t5dec_self_attention: at most %d positions (H = %d)", T5_MAX_H, H);
    return RQB_ERR_UNSUPPORTED;
  }
  const int64_t inner = (int64_t)heads * T5_DKV;
  RQB_CHECK_ARG(ldqkv >= 3 * inner && ldo >= inner && slot_stride >= (int64_t)R * inner,
                "t5dec_self_attention: a leading dimension or the slot stride is too small");
  if (R == 0) return RQB_OK;
  RQB_CHECK_ARG(qkv && cache_k && cache_v && bias && out, "t5dec_self_attention: null pointer");
  RQB_CHECK_ARG(h == 0 || (anc_in && (!parent || anc_out)), "t5dec_self_attention: h > 0 needs the ancestor table");
  const int64_t warps = (int64_t)R * heads;
  RQB_CHECK_ARG(warps <= (int64_t)INT32_MAX - 7, "t5dec_self_attention: too many rows");
  t5dec_self_attention_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      qkv, ldqkv, cache_k, cache_v, slot_stride, bias, anc_in, parent, anc_out, R, heads, h, H, out, ldo);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5dec_add_norm(float* x, const float* delta, int64_t ld_delta, const float* emb, const int64_t* ids,
                                     int64_t ids_stride, int64_t id_offset, int64_t n_emb, const float* weight, int R, int D,
                                     float eps, float* out, void* stream) {
  RQB_CHECK_ARG(R >= 0 && D > 0 && (!delta || ld_delta >= D) && (!emb || n_emb > 0), "t5dec_add_norm: bad shape (R=%d D=%d)", R,
                D);
  if (R == 0) return RQB_OK;
  RQB_CHECK_ARG(x && weight && out, "t5dec_add_norm: null pointer");
  t5dec_add_norm_kernel<<<(R + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, delta, ld_delta, emb, ids, ids_stride, id_offset, n_emb, weight, R, D, eps, out);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}
