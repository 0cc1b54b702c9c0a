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
//   rqb200_t5enc_attention  bidirectional self-attention over the packed rows, one CTA per (history, head, 128 queries), one
//                           thread per query with its q and output row in registers.  Keys and values stream through shared memory
//                           32 at a time with an online fp32 softmax, so the history length has no fixed limit.  Each score is
//                           q . k + (rel[j - i] + key_mask), HF's order; rel is HF's relative-position bias as a function of the
//                           ORIGINAL positions, so dropped positions and holes in the mask do not shift any distance.
//   rqb200_t5enc_scatter    one warp per row of the [B * S, D] output: the packed row of slot[r], or zeros for a dropped position.
//
// Numerics are HF's: no 1/sqrt(d) scaling, fp32 softmax, RMS norm in fp32.
#include <cfloat>

#include "common.cuh"

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
}

// ------------------------------------------------------------------------------------------------ self-attention
// grid (B, heads, ceil(S / TE_AQ)).  qkv row r: q at n * 64, k at inner + n * 64, v at 2 inner + n * 64.  rel [heads, 2S - 1]:
// the bias of key position pj for query position pi is rel[n, pj - pi + S - 1].
__global__ void __launch_bounds__(TE_AQ) t5enc_attention_kernel(
    const float* __restrict__ qkv, int64_t ldqkv, const int* __restrict__ src, const int* __restrict__ offsets,
    const float* __restrict__ key_mask, const float* __restrict__ rel, int S, int heads, float* __restrict__ out, int64_t ldo) {
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
  if (active) relq -= src[off + qi] - b * S;                  // relq[pj] is now the bias of key position pj
  float m = -INFINITY, l = 0.f;

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
      const float p = expf(s[j] - m_new);
      lt += p;
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
#pragma unroll
  for (int c = 0; c < TE_DKV / 4; ++c) orow[c] = make_float4(o[c].x / l, o[c].y / l, o[c].z / l, o[c].w / l);
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

extern "C" int rqb200_t5enc_assemble(const float* mask, const int64_t* ids, int64_t ids_stride, const int64_t* user_ids,
                                     int64_t user_stride, const float* item_table, int64_t n_items, const float* sep_row,
                                     const float* user_table, int64_t n_users, int64_t K, int B, int n, int H, int D,
                                     const int* offsets, const float* weight, float eps, float* x, float* out, int* src, int* slot,
                                     void* stream) {
  RQB_CHECK_ARG(B >= 0 && n >= 0 && H > 0 && n % H == 0 && D > 0 && n_items > 0 && K >= 0 && ids_stride >= n,
                "t5enc_assemble: bad shape (B=%d n=%d H=%d D=%d)", B, n, H, D);
  RQB_CHECK_ARG(!user_table == !user_ids && (!user_table || n_users > 0), "t5enc_assemble: user_ids and user_table go together");
  const int64_t S = enc_len(n, H, sep_row != nullptr, user_table != nullptr);
  RQB_CHECK_ARG(S > 0 && (int64_t)B * S <= INT32_MAX, "t5enc_assemble: bad encoder length (S=%lld, B=%d)", (long long)S, B);
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(mask && ids && item_table && offsets && weight && x && out && src && slot, "t5enc_assemble: null pointer");
  t5enc_assemble_kernel<<<B, TE_ASM, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      mask, ids, ids_stride, user_ids, user_stride, item_table, n_items, sep_row, user_table, n_users, K, n, H, (int)S, D, offsets,
      weight, eps, x, out, src, slot);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
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
  t5enc_attention_kernel<<<dim3(B, heads, tiles), TE_AQ, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      qkv, ldqkv, src, offsets, key_mask, rel, S, heads, out, ldo);
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
