// The generative-retrieval model's T5 encoder pass (transformers T5EncoderModel in eval mode, after
// EncoderDecoderRetrievalModel.encoder_forward_pass's input assembly) over the kept tokens of each history only, for
// generate(encoder="fused").  The GEMMs stay with cuBLAS and the sublayer boundaries are rqb200_t5dec_add_norm; these kernels do
// the rest:
//
//   rqb200_t5enc_offsets    one CTA: per history the number of kept positions (mask != 0; every position when none is), their
//                           exclusive scan over the batch (offsets [B + 1]: history b owns packed rows offsets[b] ..
//                           offsets[b + 1] - 1) and the additive mask of the history's keys (0, or -FLT_MAX when no position of
//                           the history is unmasked: HF then averages every position, so all of them are kept).
//   rqb200_t5enc_assemble   one CTA per history: numbers its kept positions in order, writes the packed -> (history, position)
//                           index src [N] = b * S + p and its inverse slot [B * S] (-1 for a dropped position), then one warp per
//                           kept row gathers the input row (user embedding, level-offset item id, separator) into x and writes
//                           out = T5LayerNorm(x) * weight.
//   rqb200_t5enc_assemble_capacity  the same at a fixed capacity of B * S rows (a CUDA graph cannot read N): each CTA also
//                           zeroes its share of the rows past N (x = out = 0, src = -1), which every later kernel leaves zero.
//   rqb200_t5enc_attention  bidirectional self-attention over the packed rows, one CTA per (history, head, 128 queries), one
//                           thread per query with its q and output row in registers.  Keys and values stream through shared memory
//                           32 at a time with an online fp32 softmax, so the history length has no fixed limit.  Each score is
//                           q . k + (rel[j - i] + key_mask), HF's order; rel is HF's relative-position bias as a function of the
//                           ORIGINAL positions, so dropped positions and holes in the mask do not shift any distance.
//   rqb200_t5enc_scatter    one warp per row of the [B * S, D] output: the packed row of slot[r], or zeros for a dropped position.
//
// The training pass (forward(encoder="fused")) adds:
//   rqb200_t5enc_attention_train     the attention kernel above with HF's attention-weight dropout and the row's log-sum-exp saved.
//                                    Keep bits are not stored: each is a Philox4x32-10 draw keyed on a per-call seed (read from
//                                    device memory) and counted by (history, head, query position, key position), so the backward
//                                    derives the same bits and a [B, heads, S, S] tensor never exists.
//   rqb200_t5enc_attention_backward  two launches, no global atomics: a query-major pass (D_i = dO_i . O_i, dQ and per-CTA partials
//                                    of d_rel, the relative-bias bins summed in a per-warp shared array in a fixed order) and a
//                                    key-major pass (dK and dV).  P is recomputed from the saved log-sum-exp.
//   rqb200_t5enc_dropout_keep        the keep bits of given shapes and seed, so tests can restate the forward pass.
//   rqb200_t5enc_add_norm_fwd / _bwd an out-of-place add + T5LayerNorm that saves the new residual row and its inverse RMS, and its
//                                    backward with per-CTA partials of d_weight.
//
// Numerics are HF's: no 1/sqrt(d) scaling, fp32 softmax, RMS norm in fp32.
#include <cfloat>

#include "common.cuh"
#include "t5_dropout.cuh"

#define TE_DKV 64           // d_kv, as in csrc/t5dec.cu
#define TE_SCAN 1024        // threads of the offsets kernel (histories per chunk)
#define TE_ASM 256          // threads of the assembly kernel
#define TE_AQ 128           // queries per attention CTA (one per thread)
#define TE_AK 32            // keys per shared-memory tile

// Where position p of a history sits in the encoder input: 0 user row, 1 item id (c = column of the id in the [B, n] inputs,
// j = its level), 2 separator (c = column of the item's last id).
struct EncPos {
  int kind, c, j;
};

__device__ __forceinline__ EncPos enc_pos(int p, int user, int H, int sep) {
  if (user && p == 0) return {0, 0, 0};
  const int q = p - user, W = H + sep, i = q / W, j = q % W;
  return j < H ? EncPos{1, i * H + j, j} : EncPos{2, i * H + H - 1, 0};
}

// ------------------------------------------------------------------------------------------------ offsets
__global__ void __launch_bounds__(TE_SCAN) t5enc_offsets_kernel(const float* __restrict__ mask, int B, int n, int H, int sep,
                                                                 int user, int S, int* __restrict__ offsets,
                                                                 float* __restrict__ key_mask) {
  __shared__ int cnt[TE_SCAN];
  __shared__ int wsum[TE_SCAN / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int carry = 0;
  for (int c0 = 0; c0 < B; c0 += TE_SCAN) {
    for (int i = warp; i < TE_SCAN; i += TE_SCAN / 32) {     // one warp per history: coalesced reads of its mask row
      const int b = c0 + i;
      int kept = 0;
      if (b < B) {
        const float* mr = mask + (int64_t)b * n;
        for (int c = lane; c < n; c += 32) {
          const bool on = mr[c] != 0.f;
          kept += on + (sep && c % H == H - 1 && on);
        }
        kept = __reduce_add_sync(0xffffffffu, kept) + user;
        if (lane == 0) key_mask[b] = kept ? 0.f : -FLT_MAX;
        if (kept == 0) kept = S;
      }
      if (lane == 0) cnt[i] = kept;
    }
    __syncthreads();
    const int v = cnt[threadIdx.x];
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    int before = carry, total = carry;
    for (int w = 0; w < TE_SCAN / 32; ++w) {
      if (w < warp) before += wsum[w];
      total += wsum[w];
    }
    if (c0 + threadIdx.x < B) offsets[c0 + threadIdx.x] = before + incl - v;
    carry = total;
    __syncthreads();                                          // cnt / wsum are rewritten by the next chunk
  }
  if (threadIdx.x == 0) offsets[B] = carry;
}

// ------------------------------------------------------------------------------------------------ input assembly + first norm
// CAPACITY: x, out and src hold B * S rows; history b also owns the S - cnt rows past offsets[B] that its dropped positions leave
// (starting at offsets[B] + b * S - offsets[b], so the B ranges tile offsets[B] .. B * S - 1) and writes them x = out = 0, src = -1.
template <bool CAPACITY>
__global__ void __launch_bounds__(TE_ASM) t5enc_assemble_kernel(
    const float* __restrict__ mask, const int64_t* __restrict__ ids, int64_t ids_stride, const int64_t* __restrict__ user_ids,
    int64_t user_stride, const float* __restrict__ item_table, int64_t n_items, const float* __restrict__ sep_row,
    const float* __restrict__ user_table, int64_t n_users, int64_t K, int n, int H, int S, int D, const int* __restrict__ offsets,
    const float* __restrict__ weight, float eps, float* __restrict__ x, float* __restrict__ out, int* __restrict__ src,
    int* __restrict__ slot) {
  __shared__ int wsum[TE_ASM / 32];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int user = user_table != nullptr, sep = sep_row != nullptr;
  const int off = offsets[b], cnt = offsets[b + 1] - off;
  const bool all = cnt == S;                                  // every position kept (all unmasked, or none is)
  const float* mr = mask + (int64_t)b * n;
  int base = 0;
  for (int p0 = 0; p0 < S; p0 += TE_ASM) {
    const int p = p0 + threadIdx.x;
    bool keep = false;
    if (p < S) {
      const EncPos e = enc_pos(p, user, H, sep);
      keep = all || e.kind == 0 || mr[e.c] != 0.f;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int woff = 0, total = 0;
    for (int w = 0; w < TE_ASM / 32; ++w) {
      if (w < warp) woff += wsum[w];
      total += wsum[w];
    }
    if (p < S) {
      const int r = off + base + woff + __popc(bal & ((1u << lane) - 1u));
      slot[(int64_t)b * S + p] = keep ? r : -1;
      if (keep) src[r] = b * S + p;
    }
    base += total;
    __syncthreads();                                          // wsum is rewritten by the next chunk; src is read below
  }

  for (int r = off + warp; r < off + cnt; r += TE_ASM / 32) {
    const EncPos e = enc_pos(src[r] - b * S, user, H, sep);
    const float* er;
    bool ok = true;
    if (e.kind == 0) {
      const int64_t u = user_ids[(int64_t)b * user_stride] % n_users;
      er = user_table + (u < 0 ? u + n_users : u) * D;        // torch.remainder: the sign of the divisor
    } else if (e.kind == 1) {
      const int64_t id = (ids[(int64_t)b * ids_stride + e.c] + e.j * K) * (int64_t)mr[e.c];
      ok = id >= 0 && id < n_items;
      er = item_table + (ok ? id : 0) * D;
    } else {
      er = sep_row;
    }
    float* xr = x + (int64_t)r * D;
    float ss = 0.f;
    for (int d = lane; d < D; d += 32) {
      const float val = ok ? er[d] : __int_as_float(0x7fffffff);
      xr[d] = val;
      ss = fmaf(val, val, ss);
    }
    const float inv = rsqrtf(warp_sum(ss) / (float)D + eps);
    float* orow = out + (int64_t)r * D;
    for (int d = lane; d < D; d += 32) orow[d] = weight[d] * (xr[d] * inv);
  }
  if (CAPACITY) {
    const int r0 = offsets[gridDim.x] + b * S - off;
    for (int r = r0 + warp; r < r0 + S - cnt; r += TE_ASM / 32) {
      for (int d = lane; d < D; d += 32) {
        x[(int64_t)r * D + d] = 0.f;
        out[(int64_t)r * D + d] = 0.f;
      }
      if (lane == 0) src[r] = -1;
    }
  }
}

// ------------------------------------------------------------------------------------------------ self-attention
// The attention-weight dropout's keep bits are te_keep of csrc/t5_dropout.cuh.
// grid (B, heads, ceil(S / TE_AQ)).  qkv row r: q at n * 64, k at inner + n * 64, v at 2 inner + n * 64.  rel [heads, 2S - 1]:
// the bias of key position pj for query position pi is rel[n, pj - pi + S - 1].  TRAIN adds the dropout of the attention weights
// (thresh != 0: a dropped weight leaves the sum of values, a kept one is scaled by `scale` = 1 / (1 - p); l stays the undropped
// sum) and writes lse[row * heads + n] = (m - key_mask) + log l, the log-sum-exp of the scores less key_mask (finite also for a
// history whose scores all round to -FLT_MAX).
template <bool TRAIN>
__global__ void __launch_bounds__(TE_AQ) t5enc_attention_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, const int* __restrict__ src, const int* __restrict__ offsets,
    const float* __restrict__ key_mask, const float* __restrict__ rel, int S, int heads, float* __restrict__ out, int64_t ldo,
    const int64_t* __restrict__ seed, uint32_t thresh, float scale, float* __restrict__ lse) {
  __shared__ float4 sk[TE_AK][TE_DKV / 4];
  __shared__ float4 sv[TE_AK][TE_DKV / 4];
  __shared__ int spos[TE_AK];
  const int b = blockIdx.x, n = blockIdx.y;
  const int off = offsets[b], cnt = offsets[b + 1] - off;
  const int q0 = blockIdx.z * TE_AQ;
  if (q0 >= cnt) return;                                      // uniform over the CTA
  const int qi = q0 + threadIdx.x;
  const bool active = qi < cnt;
  const int64_t inner = (int64_t)heads * TE_DKV;
  const float km = key_mask[b];
  const float* relq = rel + (int64_t)n * (2 * S - 1) + (S - 1);

  float4 q[TE_DKV / 4], o[TE_DKV / 4];
#pragma unroll
  for (int c = 0; c < TE_DKV / 4; ++c) {
    q[c] = active ? reinterpret_cast<const float4*>(qkv + (int64_t)(off + qi) * ldqkv + n * TE_DKV)[c] : make_float4(0, 0, 0, 0);
    o[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const int pi = active ? src[off + qi] - b * S : 0;
  relq -= pi;                                                 // relq[pj] is now the bias of key position pj
  float m = -INFINITY, l = 0.f;
  uint2 key = make_uint2(0u, 0u);
  if (TRAIN && thresh) key = te_seed_key(seed);

  for (int t0 = 0; t0 < cnt; t0 += TE_AK) {
    __syncthreads();                                          // the previous tile is consumed
    for (int i = threadIdx.x; i < TE_AK * TE_DKV / 4; i += TE_AQ) {
      const int j = i / (TE_DKV / 4), c = i % (TE_DKV / 4);
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (t0 + j < cnt) {
        const float* row = qkv + (int64_t)(off + t0 + j) * ldqkv + n * TE_DKV;
        kv = reinterpret_cast<const float4*>(row + inner)[c];
        vv = reinterpret_cast<const float4*>(row + 2 * inner)[c];
      }
      sk[j][c] = kv;
      sv[j][c] = vv;
    }
    if (threadIdx.x < TE_AK) spos[threadIdx.x] = t0 + (int)threadIdx.x < cnt ? src[off + t0 + threadIdx.x] - b * S : -1;
    __syncthreads();
    if (!active) continue;
    float s[TE_AK];
    float mt = -INFINITY;
    unsigned drop = 0u;                                       // bit j: key j's weight is dropped
#pragma unroll
    for (int j = 0; j < TE_AK; ++j) {
      float dot = 0.f;
#pragma unroll
      for (int c = 0; c < TE_DKV / 4; ++c) {
        const float4 k4 = sk[j][c];
        dot = fmaf(q[c].x, k4.x, dot);
        dot = fmaf(q[c].y, k4.y, dot);
        dot = fmaf(q[c].z, k4.z, dot);
        dot = fmaf(q[c].w, k4.w, dot);
      }
      const int pj = spos[j];
      s[j] = pj < 0 ? -INFINITY : dot + (relq[pj] + km);     // a key past the history contributes exp(-inf) = 0
      mt = fmaxf(mt, s[j]);
      if (TRAIN && thresh && pj >= 0 && !te_keep(key, b, n, pi, pj, thresh)) drop |= 1u << j;
    }
    const float m_new = fmaxf(m, mt);                         // finite: every tile holds at least one key of the history
    const float alpha = expf(m - m_new);
    // the tile's weighted values are summed apart and then added to the running sum: a blocked sum, so the rounding error of a
    // long, flat softmax (a fully masked history averages every position) grows with the tile and tile counts, not the length
    float4 t[TE_DKV / 4];
    float lt = 0.f;
#pragma unroll
    for (int c = 0; c < TE_DKV / 4; ++c) t[c] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < TE_AK; ++j) {
      float p = expf(s[j] - m_new);
      lt += p;
      if (TRAIN && (drop >> j & 1u)) p = 0.f;
#pragma unroll
      for (int c = 0; c < TE_DKV / 4; ++c) {
        const float4 v4 = sv[j][c];
        t[c].x = fmaf(p, v4.x, t[c].x);
        t[c].y = fmaf(p, v4.y, t[c].y);
        t[c].z = fmaf(p, v4.z, t[c].z);
        t[c].w = fmaf(p, v4.w, t[c].w);
      }
    }
    l = fmaf(l, alpha, lt);
#pragma unroll
    for (int c = 0; c < TE_DKV / 4; ++c) {
      o[c].x = fmaf(o[c].x, alpha, t[c].x);
      o[c].y = fmaf(o[c].y, alpha, t[c].y);
      o[c].z = fmaf(o[c].z, alpha, t[c].z);
      o[c].w = fmaf(o[c].w, alpha, t[c].w);
    }
    m = m_new;
  }
  if (!active) return;
  float4* orow = reinterpret_cast<float4*>(out + (int64_t)(off + qi) * ldo + n * TE_DKV);
  if (TRAIN && thresh) {
#pragma unroll
    for (int c = 0; c < TE_DKV / 4; ++c)
      orow[c] = make_float4(o[c].x / l * scale, o[c].y / l * scale, o[c].z / l * scale, o[c].w / l * scale);
  } else {
#pragma unroll
    for (int c = 0; c < TE_DKV / 4; ++c) orow[c] = make_float4(o[c].x / l, o[c].y / l, o[c].z / l, o[c].w / l);
  }
  if (TRAIN) lse[(int64_t)(off + qi) * heads + n] = (m - km) + logf(l);
}

// ------------------------------------------------------------------------------------------------ scatter
__global__ void __launch_bounds__(256) t5enc_scatter_kernel(const float* __restrict__ rows, const int* __restrict__ slot,
                                                            int64_t n_out, int D, float* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n_out) return;
  const int s = slot[r];
  const float* in = s >= 0 ? rows + (int64_t)s * D : nullptr;
  float* o = out + r * D;
  for (int d = lane; d < D; d += 32) o[d] = in ? in[d] : 0.f;
}

// ------------------------------------------------------------------------------------------------ attention backward
// Two threads per query (query-major pass) or per key (key-major pass), each holding 32 of the head's 64 dimensions; a dot product
// is the pair's two halves summed with one shuffle.  dS_ij = P_ij (dP_ij z_ij - D_i) with z_ij = keep_ij * scale, dP_ij = dO_i . v_j,
// D_i = dO_i . O_i and P_ij = exp((s_ij - key_mask) - lse_i).
#define TB_Q 64             // queries (or keys) per backward CTA
#define TB_T 32             // keys (or queries) per shared-memory tile
#define TB_W 4              // warps per backward CTA
#define TB_H (TE_DKV / 2 / 4)  // float4 per half row

__device__ __forceinline__ float half_dot(const float4* a, const float4* b) {
  float d = 0.f;
#pragma unroll
  for (int c = 0; c < TB_H; ++c) {
    const float4 y = b[c];
    d = fmaf(a[c].x, y.x, d);
    d = fmaf(a[c].y, y.y, d);
    d = fmaf(a[c].z, y.z, d);
    d = fmaf(a[c].w, y.w, d);
  }
  return d + __shfl_xor_sync(0xffffffffu, d, 1);
}

__device__ __forceinline__ void half_axpy(float4* acc, float a, const float4* x) {
#pragma unroll
  for (int c = 0; c < TB_H; ++c) {
    const float4 y = x[c];
    acc[c].x = fmaf(a, y.x, acc[c].x);
    acc[c].y = fmaf(a, y.y, acc[c].y);
    acc[c].z = fmaf(a, y.z, acc[c].z);
    acc[c].w = fmaf(a, y.w, acc[c].w);
  }
}

// grid (B, heads, ceil(S / TB_Q)), TB_W warps, dynamic smem TB_W * (2S - 1) floats (one relative-bias bin array per warp).  Writes
// delta [N, heads] (D_i), dQ into dqkv and drel_part[((b * tiles + z) * heads + n) * (2S - 1) + t] (zeros for a tile past the history).
__global__ void __launch_bounds__(TB_W * 32) t5enc_attention_bwd_q_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, const float* __restrict__ o, int64_t ldo, const float* __restrict__ dout,
    int64_t lddo, const float* __restrict__ lse, const int* __restrict__ src, const int* __restrict__ offsets,
    const float* __restrict__ key_mask, const float* __restrict__ rel, int S, int heads, const int64_t* __restrict__ seed,
    uint32_t thresh, float scale, float* __restrict__ delta, float* __restrict__ dqkv, int64_t ldd, float* __restrict__ drel_part) {
  extern __shared__ float bins[];                             // [TB_W][2S - 1]
  __shared__ float4 sk[TB_T][TE_DKV / 4];
  __shared__ float4 sv[TB_T][TE_DKV / 4];
  __shared__ int spos[TB_T];
  const int b = blockIdx.x, n = blockIdx.y, R = 2 * S - 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, h = threadIdx.x & 1;
  const int off = offsets[b], cnt = offsets[b + 1] - off;
  const int q0 = blockIdx.z * TB_Q;
  float* part = drel_part + (((int64_t)b * gridDim.z + blockIdx.z) * heads + n) * R;
  if (q0 >= cnt) {                                            // uniform over the CTA
    for (int t = threadIdx.x; t < R; t += TB_W * 32) part[t] = 0.f;
    return;
  }
  const int qi = q0 + (threadIdx.x >> 1);
  const bool active = qi < cnt;
  const int64_t inner = (int64_t)heads * TE_DKV, row = off + qi;
  const float km = key_mask[b];
  float4 q[TB_H], g[TB_H], dq[TB_H];
  float di = 0.f, li = 0.f;
  int pi = 0;
  if (active) {
    const float4* qr = reinterpret_cast<const float4*>(qkv + row * ldqkv + n * TE_DKV) + h * TB_H;
    const float4* gr = reinterpret_cast<const float4*>(dout + row * lddo + n * TE_DKV) + h * TB_H;
    const float4* orw = reinterpret_cast<const float4*>(o + row * ldo + n * TE_DKV) + h * TB_H;
#pragma unroll
    for (int c = 0; c < TB_H; ++c) {
      q[c] = qr[c];
      g[c] = gr[c];
      const float4 oc = orw[c];
      di = fmaf(g[c].x, oc.x, di);
      di = fmaf(g[c].y, oc.y, di);
      di = fmaf(g[c].z, oc.z, di);
      di = fmaf(g[c].w, oc.w, di);
    }
    li = lse[row * heads + n];
    pi = src[row] - b * S;
  } else {
#pragma unroll
    for (int c = 0; c < TB_H; ++c) q[c] = g[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  di += __shfl_xor_sync(0xffffffffu, di, 1);
  if (active && h == 0) delta[row * heads + n] = di;
#pragma unroll
  for (int c = 0; c < TB_H; ++c) dq[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float* relq = rel + (int64_t)n * R + (S - 1) - pi;
  float* wbins = bins + warp * R;
  for (int t = lane; t < R; t += 32) wbins[t] = 0.f;
  const uint2 key = thresh ? te_seed_key(seed) : make_uint2(0u, 0u);

  for (int t0 = 0; t0 < cnt; t0 += TB_T) {
    __syncthreads();                                          // the previous tile is consumed
    for (int i = threadIdx.x; i < TB_T * TE_DKV / 4; i += TB_W * 32) {
      const int j = i / (TE_DKV / 4), c = i % (TE_DKV / 4);
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (t0 + j < cnt) {
        const float* r = qkv + (int64_t)(off + t0 + j) * ldqkv + n * TE_DKV;
        kv = reinterpret_cast<const float4*>(r + inner)[c];
        vv = reinterpret_cast<const float4*>(r + 2 * inner)[c];
      }
      sk[j][c] = kv;
      sv[j][c] = vv;
    }
    if (threadIdx.x < TB_T) spos[threadIdx.x] = t0 + (int)threadIdx.x < cnt ? src[off + t0 + threadIdx.x] - b * S : -1;
    __syncthreads();
    const int nk = min(TB_T, cnt - t0);
    for (int j = 0; j < nk; ++j) {
      const int pj = spos[j];
      const float s = half_dot(q, &sk[j][h * TB_H]) + (relq[pj] + km);
      const float p = active ? expf((s - km) - li) : 0.f;
      const float z = thresh ? (te_keep(key, b, n, pi, pj, thresh) ? scale : 0.f) : 1.f;
      const float ds = p * (half_dot(g, &sv[j][h * TB_H]) * z - di);
      half_axpy(dq, ds, &sk[j][h * TB_H]);
      if (active && h == 0) wbins[pj - pi + S - 1] += ds;    // the warp's 16 queries hit 16 distinct bins
      __syncwarp();
    }
  }
  if (active) {
    float4* dr = reinterpret_cast<float4*>(dqkv + row * ldd + n * TE_DKV) + h * TB_H;
#pragma unroll
    for (int c = 0; c < TB_H; ++c) dr[c] = dq[c];
  }
  __syncthreads();
  for (int t = threadIdx.x; t < R; t += TB_W * 32) {         // the warps' bins in a fixed order
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < TB_W; ++w) acc += bins[w * R + t];
    part[t] = acc;
  }
}

// grid (B, heads, ceil(S / TB_Q)): two threads per key; writes dK and dV into dqkv.
__global__ void __launch_bounds__(TB_W * 32) t5enc_attention_bwd_kv_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, const float* __restrict__ dout, int64_t lddo, const float* __restrict__ lse,
    const float* __restrict__ delta, const int* __restrict__ src, const int* __restrict__ offsets,
    const float* __restrict__ key_mask, const float* __restrict__ rel, int S, int heads, const int64_t* __restrict__ seed,
    uint32_t thresh, float scale, float* __restrict__ dqkv, int64_t ldd) {
  __shared__ float4 sq[TB_T][TE_DKV / 4];
  __shared__ float4 sg[TB_T][TE_DKV / 4];
  __shared__ float slse[TB_T], sd[TB_T];
  __shared__ int spos[TB_T];
  const int b = blockIdx.x, n = blockIdx.y, h = threadIdx.x & 1;
  const int off = offsets[b], cnt = offsets[b + 1] - off;
  const int k0 = blockIdx.z * TB_Q;
  if (k0 >= cnt) return;                                      // uniform over the CTA
  const int kj = k0 + (threadIdx.x >> 1);
  const bool active = kj < cnt;
  const int64_t inner = (int64_t)heads * TE_DKV, row = off + kj;
  const float km = key_mask[b];
  float4 k[TB_H], v[TB_H], dk[TB_H], dv[TB_H];
  int pj = 0;
  if (active) {
    const float* r = qkv + row * ldqkv + n * TE_DKV;
#pragma unroll
    for (int c = 0; c < TB_H; ++c) {
      k[c] = reinterpret_cast<const float4*>(r + inner)[h * TB_H + c];
      v[c] = reinterpret_cast<const float4*>(r + 2 * inner)[h * TB_H + c];
    }
    pj = src[row] - b * S;
  } else {
#pragma unroll
    for (int c = 0; c < TB_H; ++c) k[c] = v[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll
  for (int c = 0; c < TB_H; ++c) dk[c] = dv[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float* relk = rel + (int64_t)n * (2 * S - 1) + (S - 1) + pj;   // relk[-pi] is the bias of query position pi
  const uint2 key = thresh ? te_seed_key(seed) : make_uint2(0u, 0u);

  for (int t0 = 0; t0 < cnt; t0 += TB_T) {
    __syncthreads();
    for (int i = threadIdx.x; i < TB_T * TE_DKV / 4; i += TB_W * 32) {
      const int j = i / (TE_DKV / 4), c = i % (TE_DKV / 4);
      float4 qv = make_float4(0.f, 0.f, 0.f, 0.f), gv = qv;
      if (t0 + j < cnt) {
        qv = reinterpret_cast<const float4*>(qkv + (int64_t)(off + t0 + j) * ldqkv + n * TE_DKV)[c];
        gv = reinterpret_cast<const float4*>(dout + (int64_t)(off + t0 + j) * lddo + n * TE_DKV)[c];
      }
      sq[j][c] = qv;
      sg[j][c] = gv;
    }
    if (threadIdx.x < TB_T) {
      const int i = t0 + threadIdx.x;
      const bool in = i < cnt;
      spos[threadIdx.x] = in ? src[off + i] - b * S : -1;
      slse[threadIdx.x] = in ? lse[(int64_t)(off + i) * heads + n] : 0.f;
      sd[threadIdx.x] = in ? delta[(int64_t)(off + i) * heads + n] : 0.f;
    }
    __syncthreads();
    const int nq = min(TB_T, cnt - t0);
    for (int i = 0; i < nq; ++i) {
      const int pi = spos[i];
      const float s = half_dot(k, &sq[i][h * TB_H]) + (relk[-pi] + km);
      const float p = active ? expf((s - km) - slse[i]) : 0.f;
      const float z = thresh ? (te_keep(key, b, n, pi, pj, thresh) ? scale : 0.f) : 1.f;
      const float ds = p * (half_dot(v, &sg[i][h * TB_H]) * z - sd[i]);
      half_axpy(dv, p * z, &sg[i][h * TB_H]);
      half_axpy(dk, ds, &sq[i][h * TB_H]);
    }
  }
  if (!active) return;
  float4* dr = reinterpret_cast<float4*>(dqkv + row * ldd + n * TE_DKV);
#pragma unroll
  for (int c = 0; c < TB_H; ++c) {
    dr[(inner >> 2) + h * TB_H + c] = dk[c];
    dr[(inner >> 1) + h * TB_H + c] = dv[c];
  }
}

// ------------------------------------------------------------------------------------------------ keep bits
__global__ void __launch_bounds__(256) t5enc_dropout_keep_kernel(const int64_t* __restrict__ seed, uint32_t thresh, int heads,
                                                                 int S, int64_t total, uint8_t* __restrict__ keep) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int pj = (int)(e % S), pi = (int)(e / S % S);
  const int64_t bn = e / ((int64_t)S * S);
  keep[e] = te_keep(te_seed_key(seed), (int)(bn / heads), (int)(bn % heads), pi, pj, thresh);
}

// ------------------------------------------------------------------------------------------------ add + T5LayerNorm for training
// One warp per row: x_out = x + delta (x when delta is null), out = weight * (x_out * inv), inv_rms = inv.
__global__ void __launch_bounds__(256) t5enc_add_norm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ delta,
                                                                 int64_t ld_delta, const float* __restrict__ weight, int R, int D,
                                                                 float eps, float* __restrict__ x_out, float* __restrict__ out,
                                                                 float* __restrict__ inv_rms) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= R) return;
  const float* xr = x + (int64_t)r * D;
  const float* dr = delta ? delta + (int64_t)r * ld_delta : nullptr;
  float* xo = x_out + (int64_t)r * D;
  float ss = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float val = dr ? xr[d] + dr[d] : xr[d];
    xo[d] = val;
    ss = fmaf(val, val, ss);
  }
  const float inv = rsqrtf(warp_sum(ss) / (float)D + eps);
  __syncwarp();
  float* orow = out + (int64_t)r * D;
  for (int d = lane; d < D; d += 32) orow[d] = weight[d] * (xo[d] * inv);
  if (lane == 0) inv_rms[r] = inv;
}

#define TN_WARPS 8
#define TN_RPW 8            // rows per warp: a CTA reduces TN_WARPS * TN_RPW rows
// dx = inv * (g w - y * mean(g w y)) + d_res with y = x_out * inv; dw_part[blockIdx.x * D + d] = sum over the CTA's rows of g y,
// summed per warp in row order, then over warps in order.  Dynamic smem TN_WARPS * D floats.
__global__ void __launch_bounds__(TN_WARPS * 32) t5enc_add_norm_bwd_kernel(
    const float* __restrict__ d_out, const float* __restrict__ d_res, const float* __restrict__ x_out,
    const float* __restrict__ inv_rms, const float* __restrict__ weight, int R, int D, float* __restrict__ dx,
    float* __restrict__ dw_part) {
  extern __shared__ float acc[];                              // [TN_WARPS][D]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* wacc = acc + warp * D;
  for (int d = lane; d < D; d += 32) wacc[d] = 0.f;
  for (int i = 0; i < TN_RPW; ++i) {
    const int r = (blockIdx.x * TN_WARPS + warp) * TN_RPW + i;
    if (r >= R) break;
    const float* gr = d_out + (int64_t)r * D;
    const float* xr = x_out + (int64_t)r * D;
    const float inv = inv_rms[r];
    float dot = 0.f;
    for (int d = lane; d < D; d += 32) {
      const float y = xr[d] * inv;
      dot = fmaf(gr[d] * weight[d], y, dot);
      wacc[d] = fmaf(gr[d], y, wacc[d]);
    }
    const float c = warp_sum(dot) / (float)D;
    const float* rr = d_res ? d_res + (int64_t)r * D : nullptr;
    float* o = dx + (int64_t)r * D;
    for (int d = lane; d < D; d += 32) {
      const float y = xr[d] * inv;
      const float v = inv * (gr[d] * weight[d] - y * c);
      o[d] = rr ? v + rr[d] : v;
    }
  }
  __syncthreads();
  for (int d = threadIdx.x; d < D; d += TN_WARPS * 32) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < TN_WARPS; ++w) s += acc[w * D + d];
    dw_part[(int64_t)blockIdx.x * D + d] = s;
  }
}

// ------------------------------------------------------------------------------------------------ C ABI
static int enc_len(int n, int H, int sep, int user) { return user + n / H * (H + sep); }

extern "C" int rqb200_t5enc_offsets(const float* mask, int B, int n, int H, int sep, int user, int* offsets, float* key_mask,
                                    void* stream) {
  RQB_CHECK_ARG(B >= 0 && n >= 0 && H > 0 && n % H == 0 && (sep == 0 || sep == 1) && (user == 0 || user == 1),
                "t5enc_offsets: bad shape (B=%d n=%d H=%d sep=%d user=%d)", B, n, H, sep, user);
  const int64_t S = enc_len(n, H, sep, user);
  RQB_CHECK_ARG(S > 0, "t5enc_offsets: empty encoder sequence");
  RQB_CHECK_ARG((int64_t)B * S <= INT32_MAX, "t5enc_offsets: B * S = %lld positions exceed the int32 index",
                (long long)((int64_t)B * S));
  RQB_CHECK_ARG(offsets && (B == 0 || (mask && key_mask)), "t5enc_offsets: null pointer");
  t5enc_offsets_kernel<<<1, TE_SCAN, 0, reinterpret_cast<cudaStream_t>(stream)>>>(mask, B, n, H, sep, user, (int)S, offsets,
                                                                                   key_mask);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

template <bool CAPACITY>
static int t5enc_assemble_launch(const char* what, const float* mask, const int64_t* ids, int64_t ids_stride,
                                 const int64_t* user_ids, int64_t user_stride, const float* item_table, int64_t n_items,
                                 const float* sep_row, const float* user_table, int64_t n_users, int64_t K, int B, int n, int H, int D,
                                 const int* offsets, const float* weight, float eps, float* x, float* out, int* src, int* slot,
                                 void* stream) {
  RQB_CHECK_ARG(B >= 0 && n >= 0 && H > 0 && n % H == 0 && D > 0 && n_items > 0 && K >= 0 && ids_stride >= n,
                "%s: bad shape (B=%d n=%d H=%d D=%d)", what, B, n, H, D);
  RQB_CHECK_ARG(!user_table == !user_ids && (!user_table || n_users > 0), "%s: user_ids and user_table go together", what);
  const int64_t S = enc_len(n, H, sep_row != nullptr, user_table != nullptr);
  RQB_CHECK_ARG(S > 0 && (int64_t)B * S <= INT32_MAX, "%s: bad encoder length (S=%lld, B=%d)", what, (long long)S, B);
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(mask && ids && item_table && offsets && weight && x && out && src && slot, "%s: null pointer", what);
  t5enc_assemble_kernel<CAPACITY><<<B, TE_ASM, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      mask, ids, ids_stride, user_ids, user_stride, item_table, n_items, sep_row, user_table, n_users, K, n, H, (int)S, D, offsets,
      weight, eps, x, out, src, slot);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5enc_assemble(const float* mask, const int64_t* ids, int64_t ids_stride, const int64_t* user_ids,
                                     int64_t user_stride, const float* item_table, int64_t n_items, const float* sep_row,
                                     const float* user_table, int64_t n_users, int64_t K, int B, int n, int H, int D,
                                     const int* offsets, const float* weight, float eps, float* x, float* out, int* src, int* slot,
                                     void* stream) {
  return t5enc_assemble_launch<false>("t5enc_assemble", mask, ids, ids_stride, user_ids, user_stride, item_table, n_items,
                                      sep_row, user_table, n_users, K, B, n, H, D, offsets, weight, eps, x, out, src, slot, stream);
}

extern "C" int rqb200_t5enc_assemble_capacity(const float* mask, const int64_t* ids, int64_t ids_stride, const int64_t* user_ids,
                                              int64_t user_stride, const float* item_table, int64_t n_items, const float* sep_row,
                                              const float* user_table, int64_t n_users, int64_t K, int B, int n, int H, int D,
                                              const int* offsets, const float* weight, float eps, float* x, float* out, int* src,
                                              int* slot, void* stream) {
  return t5enc_assemble_launch<true>("t5enc_assemble_capacity", mask, ids, ids_stride, user_ids, user_stride, item_table, n_items,
                                     sep_row, user_table, n_users, K, B, n, H, D, offsets, weight, eps, x, out, src, slot, stream);
}

extern "C" int rqb200_t5enc_attention(const float* qkv, int64_t ldqkv, const int* src, const int* offsets, const float* key_mask,
                                      const float* rel, int B, int S, int heads, float* out, int64_t ldo, void* stream) {
  RQB_CHECK_ARG(B >= 0 && S > 0 && heads > 0, "t5enc_attention: bad shape (B=%d S=%d heads=%d)", B, S, heads);
  const int64_t inner = (int64_t)heads * TE_DKV;
  RQB_CHECK_ARG(ldqkv >= 3 * inner && ldo >= inner && ldqkv % 4 == 0 && ldo % 4 == 0,
                "t5enc_attention: leading dimensions must be multiples of 4, ldqkv >= 3 * heads * 64 and ldo >= heads * 64");
  RQB_CHECK_ARG(heads <= 65535 && (int64_t)B * S <= INT32_MAX, "t5enc_attention: too many heads or positions");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(qkv && src && offsets && key_mask && rel && out, "t5enc_attention: null pointer");
  RQB_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) % 16 == 0,
                "t5enc_attention: qkv and out must be 16-byte aligned");
  const unsigned tiles = (unsigned)((S + TE_AQ - 1) / TE_AQ);
  t5enc_attention_kernel<false><<<dim3(B, heads, tiles), TE_AQ, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      qkv, ldqkv, src, offsets, key_mask, rel, S, heads, out, ldo, nullptr, 0u, 1.f, nullptr);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5enc_scatter(const float* rows, const int* slot, int64_t n_out, int D, float* out, void* stream) {
  RQB_CHECK_ARG(n_out >= 0 && D > 0, "t5enc_scatter: bad shape (n_out=%lld D=%d)", (long long)n_out, D);
  if (n_out == 0) return RQB_OK;
  RQB_CHECK_ARG(rows && slot && out, "t5enc_scatter: null pointer");
  const int64_t blocks = (n_out + 7) / 8;
  RQB_CHECK_ARG(blocks <= INT32_MAX, "t5enc_scatter: too many rows");
  t5enc_scatter_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(rows, slot, n_out, D, out);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

static int attention_train_args(const float* qkv, int64_t ldqkv, int B, int S, int heads, float p, const char* what) {
  RQB_CHECK_ARG(B >= 0 && S > 0 && heads > 0, "%s: bad shape (B=%d S=%d heads=%d)", what, B, S, heads);
  RQB_CHECK_ARG(p >= 0.f && p < 1.f, "%s: dropout probability %g outside [0, 1)", what, (double)p);
  RQB_CHECK_ARG(ldqkv >= 3 * (int64_t)heads * TE_DKV && ldqkv % 4 == 0 && reinterpret_cast<uintptr_t>(qkv) % 16 == 0,
                "%s: qkv needs a row stride >= 3 * heads * 64 that is a multiple of 4 and 16-byte alignment", what);
  RQB_CHECK_ARG(heads <= 65535 && (int64_t)B * S <= INT32_MAX, "%s: too many heads or positions", what);
  return RQB_OK;
}

extern "C" int rqb200_t5enc_attention_train(const float* qkv, int64_t ldqkv, const int* src, const int* offsets,
                                            const float* key_mask, const float* rel, int B, int S, int heads, const int64_t* seed,
                                            float p, float* out, int64_t ldo, float* lse, void* stream) {
  if (int rc = attention_train_args(qkv, ldqkv, B, S, heads, p, "t5enc_attention_train")) return rc;
  RQB_CHECK_ARG(ldo >= (int64_t)heads * TE_DKV && ldo % 4 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0,
                "t5enc_attention_train: out needs a row stride >= heads * 64 that is a multiple of 4 and 16-byte alignment");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(qkv && src && offsets && key_mask && rel && out && lse && seed, "t5enc_attention_train: null pointer");
  uint32_t thresh;
  float scale;
  dropout_params(p, &thresh, &scale);
  const unsigned tiles = (unsigned)((S + TE_AQ - 1) / TE_AQ);
  t5enc_attention_kernel<true><<<dim3(B, heads, tiles), TE_AQ, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      qkv, ldqkv, src, offsets, key_mask, rel, S, heads, out, ldo, seed, thresh, scale, lse);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5enc_attention_backward_tiles(int S) { return S > 0 ? (S + TB_Q - 1) / TB_Q : 0; }

extern "C" int rqb200_t5enc_attention_backward(const float* qkv, int64_t ldqkv, const float* out, int64_t ldo, const float* dout,
                                               int64_t lddo, const float* lse, const int* src, const int* offsets,
                                               const float* key_mask, const float* rel, int B, int S, int heads,
                                               const int64_t* seed, float p, float* delta, float* dqkv, int64_t ldd,
                                               float* drel_part, void* stream) {
  if (int rc = attention_train_args(qkv, ldqkv, B, S, heads, p, "t5enc_attention_backward")) return rc;
  const int64_t inner = (int64_t)heads * TE_DKV;
  RQB_CHECK_ARG(ldo >= inner && lddo >= inner && ldd >= 3 * inner && ldo % 4 == 0 && lddo % 4 == 0 && ldd % 4 == 0 &&
                    ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(dout) | reinterpret_cast<uintptr_t>(dqkv)) %
                     16) == 0,
                "t5enc_attention_backward: out / dout need row strides >= heads * 64, dqkv >= 3 * heads * 64, all multiples of "
                "4, and 16-byte alignment");
  const size_t smem = (size_t)TB_W * (2 * S - 1) * sizeof(float);
  RQB_CHECK_ARG(smem <= 160 * 1024, "t5enc_attention_backward: S = %d positions exceed the relative-bias bins' shared memory "
                "(at most %d)", S, (160 * 1024 / (int)sizeof(float) / TB_W + 1) / 2);
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(qkv && out && dout && lse && src && offsets && key_mask && rel && seed && delta && dqkv && drel_part,
                "t5enc_attention_backward: null pointer");
  uint32_t thresh;
  float scale;
  dropout_params(p, &thresh, &scale);
  const dim3 grid(B, heads, (unsigned)rqb200_t5enc_attention_backward_tiles(S));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (smem > 48 * 1024)
    RQB_CUDA(cudaFuncSetAttribute(t5enc_attention_bwd_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  t5enc_attention_bwd_q_kernel<<<grid, TB_W * 32, smem, st>>>(qkv, ldqkv, out, ldo, dout, lddo, lse, src, offsets, key_mask, rel,
                                                              S, heads, seed, thresh, scale, delta, dqkv, ldd, drel_part);
  RQB_LAUNCH_CHECK();
  t5enc_attention_bwd_kv_kernel<<<grid, TB_W * 32, 0, st>>>(qkv, ldqkv, dout, lddo, lse, delta, src, offsets, key_mask, rel, S,
                                                            heads, seed, thresh, scale, dqkv, ldd);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5enc_dropout_keep(const int64_t* seed, float p, int B, int heads, int S, uint8_t* keep, void* stream) {
  RQB_CHECK_ARG(B >= 0 && heads > 0 && S > 0, "t5enc_dropout_keep: bad shape (B=%d heads=%d S=%d)", B, heads, S);
  RQB_CHECK_ARG(p >= 0.f && p < 1.f, "t5enc_dropout_keep: dropout probability %g outside [0, 1)", (double)p);
  const int64_t total = (int64_t)B * heads * S * S;
  if (total == 0) return RQB_OK;
  RQB_CHECK_ARG(seed && keep, "t5enc_dropout_keep: null pointer");
  RQB_CHECK_ARG((total + 255) / 256 <= INT32_MAX, "t5enc_dropout_keep: too many elements");
  uint32_t thresh;
  float scale;
  dropout_params(p, &thresh, &scale);
  t5enc_dropout_keep_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      seed, thresh, heads, S, total, keep);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5enc_add_norm_fwd(const float* x, const float* delta, int64_t ld_delta, const float* weight, int R, int D,
                                         float eps, float* x_out, float* out, float* inv_rms, void* stream) {
  RQB_CHECK_ARG(R >= 0 && D > 0 && (!delta || ld_delta >= D), "t5enc_add_norm_fwd: bad shape (R=%d D=%d)", R, D);
  if (R == 0) return RQB_OK;
  RQB_CHECK_ARG(x && weight && x_out && out && inv_rms, "t5enc_add_norm_fwd: null pointer");
  t5enc_add_norm_fwd_kernel<<<(R + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, delta, ld_delta, weight, R, D, eps,
                                                                                              x_out, out, inv_rms);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_t5enc_add_norm_bwd_parts(int R) { return R > 0 ? (R + TN_WARPS * TN_RPW - 1) / (TN_WARPS * TN_RPW) : 0; }

extern "C" int rqb200_t5enc_add_norm_bwd(const float* d_out, const float* d_res, const float* x_out, const float* inv_rms,
                                         const float* weight, int R, int D, float* dx, float* dw_part, void* stream) {
  RQB_CHECK_ARG(R >= 0 && D > 0, "t5enc_add_norm_bwd: bad shape (R=%d D=%d)", R, D);
  const size_t smem = (size_t)TN_WARPS * D * sizeof(float);
  RQB_CHECK_ARG(smem <= 160 * 1024, "t5enc_add_norm_bwd: D = %d exceeds the shared-memory accumulators", D);
  if (R == 0) return RQB_OK;
  RQB_CHECK_ARG(d_out && x_out && inv_rms && weight && dx && dw_part, "t5enc_add_norm_bwd: null pointer");
  if (smem > 48 * 1024)
    RQB_CUDA(cudaFuncSetAttribute(t5enc_add_norm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  t5enc_add_norm_bwd_kernel<<<(unsigned)rqb200_t5enc_add_norm_bwd_parts(R), TN_WARPS * 32, smem,
                              reinterpret_cast<cudaStream_t>(stream)>>>(d_out, d_res, x_out, inv_rms, weight, R, D, dx, dw_part);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}
