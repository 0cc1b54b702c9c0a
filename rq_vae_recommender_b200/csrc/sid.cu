// Corpus-side kernels of the semantic-id table (SURVEY 8(f)-1 / 8(f)-2 / the prefix check of 8(f)-4): the formats either side of the tokeniser.
//
//   rqb200_sid_dedup_rank   modules/tokenizer/semids.py:94-108: for every corpus row, how many EARLIER rows carry the identical
//                           id tuple (the reference's O(N^2) compare, 90-97 % of its corpus pass), plus the diversity statistics
//                           of train_rqvae.py:276-283 (max duplicates, number of distinct tuples, entropy of the tuple
//                           distribution) from the same pass.
//   rqb200_sid_gather       semids.py:112-146: cached_ids[item_ids] -> [B, S * C] token rows with -1 under the padding mask, and
//                           the matching token_type_ids, in one launch.
//
// Dedup without a sort: the packed tuple (K^L <= 2^26 keys: 24 bits for K = 256, L = 3) addresses a head table; pass 1 threads
// every row onto its key's list with one atomicExch; pass 2 walks the (short) list of the row's key and counts the members with
// a smaller row index.  Work is sum over keys of (group size)^2, i.e. O(N) for the near-unique tables a trained model produces,
// and never worse than the reference's O(N^2).
#include "common.cuh"

#define SID_MAX_KEYS (1ll << 26)

static int64_t sid_key_space(int L, int K) {
  int64_t s = 1;
  for (int l = 0; l < L; ++l) {
    s *= K;
    if (s > SID_MAX_KEYS) return 0;
  }
  return s;
}

extern "C" size_t rqb200_sid_dedup_workspace_bytes(int N, int L, int K) {
  const int64_t keys = sid_key_space(L, K);
  if (keys == 0 || N < 0) return 0;                      // key space too large for a direct table: the caller sorts instead
  return (size_t)(keys + N) * sizeof(int) + 64;
}

__device__ __forceinline__ int64_t sid_pack(const int64_t* row, int L, int K, bool& ok) {
  int64_t key = 0;
  ok = true;
  for (int l = 0; l < L; ++l) {
    const int64_t v = row[l];
    ok = ok && v >= 0 && v < K;
    key = key * K + v;
  }
  return key;
}

__global__ void sid_link_kernel(const int64_t* ids, int N, int L, int K, int* head, int* next) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
    bool ok;
    const int64_t key = sid_pack(ids + (int64_t)i * L, L, K, ok);
    next[i] = ok ? atomicExch(&head[key], i) : -2;       // -2: an id outside [0, K): the row is its own group
  }
}

// stats: [0] max rank, [1] distinct tuples; entropy: -sum p log p over distinct tuples (p = group size / N)
__global__ void sid_rank_kernel(const int64_t* ids, int N, int L, int K, const int* head, const int* next, int64_t* rank,
                                int* stats, double* entropy) {
  double ent = 0.0;
  int mx = 0, uniq = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
    int r = 0, g = 1;
    if (next[i] != -2) {
      bool ok;
      const int64_t key = sid_pack(ids + (int64_t)i * L, L, K, ok);
      g = 0;
      for (int j = head[key]; j >= 0; j = next[j]) {     // the list holds exactly the rows with this key
        r += (j < i);
        ++g;
      }
    }
    rank[i] = r;
    mx = max(mx, r);
    if (r == 0) {                                        // the earliest row of its group speaks for the group
      ++uniq;
      const double p = (double)g / (double)N;
      ent -= p * log(p);
    }
  }
  ent = warp_sum_d(ent);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    uniq += __shfl_xor_sync(0xffffffffu, uniq, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(&stats[0], mx);
    atomicAdd(&stats[1], uniq);
    atomicAdd(entropy, ent);
  }
}

extern "C" int rqb200_sid_dedup_rank(const int64_t* ids, int N, int L, int K, int64_t* rank, int* stats, double* entropy,
                                     void* workspace, size_t ws_bytes, void* stream) {
  const int64_t keys = sid_key_space(L, K);
  if (keys == 0) {
    rqb_set_error("sid_dedup_rank: key space K^L = %d^%d exceeds the direct table (2^26 keys)", K, L);
    return RQB_ERR_UNSUPPORTED;
  }
  RQB_CHECK_ARG(N >= 0 && L > 0 && K > 0 && stats && entropy, "sid_dedup_rank: bad argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RQB_CUDA(cudaMemsetAsync(stats, 0, 2 * sizeof(int), st));
  RQB_CUDA(cudaMemsetAsync(entropy, 0, sizeof(double), st));
  if (N == 0) return RQB_OK;
  RQB_CHECK_ARG(ids && rank && workspace, "sid_dedup_rank: null pointer");
  if (ws_bytes < rqb200_sid_dedup_workspace_bytes(N, L, K)) {
    rqb_set_error("sid_dedup_rank: workspace too small");
    return RQB_ERR_WORKSPACE;
  }
  int* head = reinterpret_cast<int*>(workspace);
  int* next = head + keys;
  RQB_CUDA(cudaMemsetAsync(head, 0xFF, (size_t)keys * sizeof(int), st));     // -1 = empty list
  int grid = (N + 255) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  sid_link_kernel<<<grid, 256, 0, st>>>(ids, N, L, K, head, next);
  RQB_LAUNCH_CHECK();
  sid_rank_kernel<<<grid, 256, 0, st>>>(ids, N, L, K, head, next, rank, stats, entropy);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// out[b, s * C + c] = mask[b, s] ? cached[item[b, s], c] : -1;   token_type[b, s * C + c] = c     (mask may be null: all valid)
__global__ void sid_gather_kernel(const int64_t* __restrict__ cached, int C, const int64_t* __restrict__ item, int64_t item_stride,
                                  const unsigned char* __restrict__ mask, int64_t mask_stride, int B, int S, int64_t* __restrict__ out,
                                  int64_t* __restrict__ token_type) {
  const int64_t total = (int64_t)B * S * C;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(e % C);
    const int64_t bs = e / C;
    const int s = (int)(bs % S);
    const int64_t b = bs / S;
    const bool valid = mask == nullptr || mask[b * mask_stride + s] != 0;
    int64_t v = -1;
    if (valid) v = cached[item[b * item_stride + s] * C + c];
    out[e] = v;
    if (token_type) token_type[e] = c;
  }
}

extern "C" int rqb200_sid_gather(const int64_t* cached_ids, int64_t n_corpus, int C, const int64_t* item_ids, int64_t item_stride,
                                 const unsigned char* seq_mask, int64_t mask_stride, int B, int S, int64_t* out,
                                 int64_t* token_type, void* stream) {
  RQB_CHECK_ARG(B >= 0 && S >= 0 && C > 0 && n_corpus >= 0, "sid_gather: bad shape");
  if ((int64_t)B * S == 0) return RQB_OK;
  RQB_CHECK_ARG(cached_ids && item_ids && out, "sid_gather: null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t total = (int64_t)B * S * C;
  int grid = (int)((total + 255) / 256);
  if (grid > 132 * 8) grid = 132 * 8;
  sid_gather_kernel<<<grid, 256, 0, st>>>(cached_ids, C, item_ids, item_stride, seq_mask, mask_stride, B, S, out, token_type);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Valid-prefix index of the corpus id table (SURVEY 8(f)-4: modules/model.py:169-182 `_check_valid_prefix`, called once per
// hierarchy level of the constrained beam search, :340-376).  The reference compares every candidate prefix with every corpus
// row: O(P N l) per call (P = batch x beams x candidates = 163 840 at the shipped evaluation settings, N = corpus size).  Here
// the corpus is turned ONCE into one bitmap per prefix length l (bit key = packed prefix, K^l bits: 32 B, 8 KB, 2 MB, 512 MB for
// K = 256, l = 1..4) and a check is one bit test per prefix.
//   workspace layout: for l = 1..C the bitmap of ceil(K^l / 32) words, each region padded to 256 bytes, in this order.
#define SID_PREFIX_MAX_BITS (1ll << 33)

static int64_t sid_prefix_bits(int l, int K) {
  int64_t s = 1;
  for (int i = 0; i < l; ++i) {
    s *= K;
    if (s > SID_PREFIX_MAX_BITS) return 0;
  }
  return s;
}
static size_t sid_prefix_region(int l, int K) {            // bytes of level l's bitmap region (0: too large)
  const int64_t bits = sid_prefix_bits(l, K);
  if (bits == 0) return 0;
  return (size_t)(((bits + 31) / 32 * 4 + 255) / 256 * 256);
}

extern "C" size_t rqb200_sid_prefix_workspace_bytes(int C, int K) {
  if (C <= 0 || C > 8 || K <= 0) return 0;
  size_t tot = 0;
  for (int l = 1; l <= C; ++l) {
    const size_t r = sid_prefix_region(l, K);
    if (r == 0) return 0;                                   // key space too large for bitmaps: the caller keeps the reference's compare
    tot += r;
  }
  return tot;
}

struct SidPrefixOffsets { unsigned long long off[9]; };     // off[l] = byte offset of level l's bitmap (1-based)

__global__ void sid_prefix_build_kernel(const int64_t* __restrict__ ids, int64_t N, int C, int K, unsigned int* ws, SidPrefixOffsets o) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
    unsigned long long key = 0;
    for (int l = 1; l <= C; ++l) {
      const int64_t v = ids[i * C + l - 1];
      if (v < 0 || v >= K) break;                           // an id outside [0, K) can never equal a candidate drawn from K logits
      key = key * (unsigned long long)K + (unsigned long long)v;
      atomicOr(ws + o.off[l] / 4 + (key >> 5), 1u << (key & 31));
    }
  }
}

// valid[p] = any corpus row whose first l ids equal prefix[p, :l]      (model.py:175-181)
__global__ void sid_prefix_check_kernel(const int64_t* __restrict__ prefix, int64_t stride, int64_t P, int l, int K,
                                        const unsigned int* __restrict__ bitmap, unsigned char* __restrict__ valid) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (int64_t)gridDim.x * blockDim.x) {
    unsigned long long key = 0;
    bool ok = true;
    for (int j = 0; j < l; ++j) {
      const int64_t v = prefix[p * stride + j];
      ok = ok && v >= 0 && v < K;
      key = key * (unsigned long long)K + (unsigned long long)(ok ? v : 0);
    }
    valid[p] = (ok && ((__ldg(bitmap + (key >> 5)) >> (key & 31)) & 1u)) ? 1 : 0;
  }
}

static int sid_prefix_offsets(int C, int K, SidPrefixOffsets& o) {
  size_t at = 0;
  for (int l = 1; l <= C; ++l) {
    const size_t r = sid_prefix_region(l, K);
    if (r == 0) return 1;
    o.off[l] = at;
    at += r;
  }
  return 0;
}

extern "C" int rqb200_sid_prefix_build(const int64_t* cached_ids, int64_t N, int C, int K, void* workspace, size_t ws_bytes, void* stream) {
  RQB_CHECK_ARG(N >= 0 && C > 0 && C <= 8 && K > 0 && workspace, "sid_prefix_build: bad argument");
  const size_t need = rqb200_sid_prefix_workspace_bytes(C, K);
  if (need == 0) {
    rqb_set_error("sid_prefix_build: key space K^C = %d^%d exceeds the bitmap limit (2^33 bits)", K, C);
    return RQB_ERR_UNSUPPORTED;
  }
  if (ws_bytes < need) {
    rqb_set_error("sid_prefix_build: workspace too small");
    return RQB_ERR_WORKSPACE;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RQB_CUDA(cudaMemsetAsync(workspace, 0, need, st));
  if (N == 0) return RQB_OK;
  RQB_CHECK_ARG(cached_ids, "sid_prefix_build: null pointer");
  SidPrefixOffsets o{};
  sid_prefix_offsets(C, K, o);
  int grid = (int)((N + 255) / 256);
  if (grid > 132 * 8) grid = 132 * 8;
  sid_prefix_build_kernel<<<grid, 256, 0, st>>>(cached_ids, N, C, K, reinterpret_cast<unsigned int*>(workspace), o);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_sid_prefix_check(const int64_t* prefix, int64_t row_stride, int64_t P, int l, int C, int K, const void* workspace,
                                       unsigned char* valid, void* stream) {
  RQB_CHECK_ARG(P >= 0 && l > 0 && l <= C && C <= 8 && K > 0 && row_stride >= l, "sid_prefix_check: bad argument (l=%d C=%d)", l, C);
  if (P == 0) return RQB_OK;
  RQB_CHECK_ARG(prefix && workspace && valid, "sid_prefix_check: null pointer");
  SidPrefixOffsets o{};
  if (sid_prefix_offsets(C, K, o)) {
    rqb_set_error("sid_prefix_check: key space too large");
    return RQB_ERR_UNSUPPORTED;
  }
  int grid = (int)((P + 255) / 256);
  if (grid > 132 * 16) grid = 132 * 16;
  sid_prefix_check_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      prefix, row_stride, P, l, K, reinterpret_cast<const unsigned int*>(reinterpret_cast<const char*>(workspace) + o.off[l]), valid);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// One selection step of the constrained beam search (modules/model.py:340-376) in one launch: for every batch row the
// kp x nc candidate extensions (kp live beams, nc sampled tokens each) are scored  log p(token) + log p(parent beam),  the
// extensions whose id prefix does not occur in the corpus get -inf (bit test in the prefix index above: the reference's
// repeat_interleave + cat + O(P N) compare + masked_fill), and the k best are taken in descending score order (the reference
// sorts all kp nc scores and keeps k), with their ids gathered into the new beams and the parent beam's global index returned
// for the key/value-cache reorder.  Ties: lowest flat candidate index first (torch.sort is not stable: any order is legal).
// One warp per batch row; kp * nc <= 1024, k <= 32.
#define SID_BEAM_MAX_E 1024

__global__ void __launch_bounds__(128) sid_beam_select_kernel(
    const int64_t* __restrict__ samples, const float* __restrict__ samp_log_p, const int64_t* __restrict__ generated,
    const float* __restrict__ log_probas, int B, int kp, int nc, int h, int k, int K, const unsigned int* __restrict__ bitmap,
    int64_t* __restrict__ out_generated, float* __restrict__ out_log_probas, int64_t* __restrict__ out_parent) {
  __shared__ float s_score[4][SID_BEAM_MAX_E];
  __shared__ unsigned char s_taken[4][SID_BEAM_MAX_E];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * 4 + w;
  if (b >= B) return;
  const int E = kp * nc;
  float* sc = s_score[w];
  unsigned char* tk = s_taken[w];
  for (int e = lane; e < E; e += 32) {
    const int beam = e / nc;
    const int64_t tok = samples[((int64_t)b * kp + beam) * nc + (e - beam * nc)];
    unsigned long long key = 0;
    bool ok = tok >= 0 && tok < K;
    for (int j = 0; j < h; ++j) {
      const int64_t v = generated[((int64_t)b * kp + beam) * h + j];
      ok = ok && v >= 0 && v < K;
      key = key * (unsigned long long)K + (unsigned long long)(ok ? v : 0);
    }
    key = key * (unsigned long long)K + (unsigned long long)(ok ? tok : 0);
    ok = ok && ((__ldg(bitmap + (key >> 5)) >> (key & 31)) & 1u);
    float s = samp_log_p[((int64_t)b * kp + beam) * nc + (e - beam * nc)] + (log_probas ? log_probas[(int64_t)b * kp + beam] : 0.f);
    if (!ok || s != s) s = -INFINITY;                       // invalid prefix (model.py:356,366); NaN ranks last here
    sc[e] = s;
    tk[e] = 0;
  }
  __syncwarp();
  for (int r = 0; r < k; ++r) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int e = lane; e < E; e += 32) {
      if (tk[e]) continue;
      const float s = sc[e];
      if (s > best || bi == 0x7fffffff) { best = s; bi = e; }            // ascending e per lane: the first maximum stays
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi != 0x7fffffff && (bi == 0x7fffffff || ob > best || (ob == best && oi < bi))) { best = ob; bi = oi; }
    }
    if (bi == 0x7fffffff) { bi = 0; best = -INFINITY; }     // k > kp * nc: repeat entry 0 with -inf (the reference would fail)
    const int beam = bi / nc;
    if (lane == 0) {
      tk[bi] = 1;
      out_log_probas[(int64_t)b * k + r] = best;
      out_parent[(int64_t)b * k + r] = (int64_t)b * kp + beam;
      out_generated[((int64_t)b * k + r) * (h + 1) + h] = samples[((int64_t)b * kp + beam) * nc + (bi - beam * nc)];
    }
    for (int j = lane; j < h; j += 32)
      out_generated[((int64_t)b * k + r) * (h + 1) + j] = generated[((int64_t)b * kp + beam) * h + j];
    __syncwarp();
  }
}

extern "C" int rqb200_sid_beam_select(const int64_t* samples, const float* samp_log_p, const int64_t* generated,
                                      const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K,
                                      const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                      int64_t* out_parent, void* stream) {
  RQB_CHECK_ARG(B >= 0 && kp > 0 && nc > 0 && h >= 0 && h < C && C <= 8 && k > 0 && K > 0, "sid_beam_select: bad argument");
  if (kp * nc > SID_BEAM_MAX_E || k > 32) {
    rqb_set_error("sid_beam_select: kp * nc = %d (max %d), k = %d (max 32)", kp * nc, SID_BEAM_MAX_E, k);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(samples && samp_log_p && prefix_workspace && out_generated && out_log_probas && out_parent && (h == 0 || generated),
                "sid_beam_select: null pointer");
  SidPrefixOffsets o{};
  if (sid_prefix_offsets(C, K, o)) {
    rqb_set_error("sid_beam_select: key space too large");
    return RQB_ERR_UNSUPPORTED;
  }
  sid_beam_select_kernel<<<(B + 3) / 4, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      samples, samp_log_p, generated, log_probas, B, kp, nc, h, k, K,
      reinterpret_cast<const unsigned int*>(reinterpret_cast<const char*>(prefix_workspace) + o.off[h + 1]), out_generated,
      out_log_probas, out_parent);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}
