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
#include <utility>

#include <cub/block/block_radix_sort.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "sid_excl.cuh"

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
// the corpus is turned ONCE into a trie of its distinct prefixes, O(N C) bytes for any K^C, which the search kernels below
// read.  It holds exactly the prefixes of the corpus rows up to their first id outside [0, K): a prefix holding such an id is
// never valid (it can never equal a candidate drawn from K logits).
//
// Level l (1..C) holds the n[l] distinct l-prefixes of the corpus rows in lexicographic order; node i of level l
// stores its last code code_l[i] and, for l < C, the range of its children in level l + 1, [child_l[i], child_l[i + 1]) (the
// root is level 0: child_0 = {0, n[1]}).  Lexicographic order makes the children of a node contiguous and sorted by code, so
// "node i extended by code c" is a binary search in at most K codes.  The workspace starts with a SidTrieHeader that locates
// the arrays, so a search call needs only the workspace pointer.
//   workspace layout: header | child_0 .. child_{C-1} (int [cap_l + 1]) | code_1 .. code_C (uint16 [N]), every region
//   256-byte aligned, cap_0 = 1 and cap_l = N (a level has at most N nodes).  The build's sort scratch (SidSortScratch) is a
//   separate buffer, needed only while the build runs.
// Build: rows are sorted lexicographically (stable LSD radix sort over 64-bit keys of as many columns as fit, ids outside
// [0, K) and every id after them mapped to K so that they sort last), each sorted row flags the levels at which it starts a new
// node (deeper than its common prefix with the row before, within its valid length), an inclusive scan per level numbers the
// nodes, and one pass writes codes and child ranges.
struct SidTrieHeader {
  int C, K;
  long long N;
  int n[9];                                                 // nodes per level; n[0] = 1 (the root)
  unsigned long long child[8];                              // byte offset of child_l, l = 0..C-1
  unsigned long long code[9];                               // byte offset of code_l, l = 1..C
};

static size_t sid_align256(size_t b) { return (b + 255) / 256 * 256; }

// bits per id in the packed sort keys of the trie and the item table (K itself, the "no id" mark, fits); 64 / width ids fit
// one 64-bit key
static int sid_id_bits(int K) { return 32 - __builtin_clz((unsigned)K); }

// Scratch of the row sort shared by the trie and the item table, as byte offsets: two buffers of 64-bit sort keys and two of
// row permutations (N each), `levels` arrays of N ints for the flags and as many for their scans, and CUB's temp storage for a
// sort or a scan of N entries.
struct SidSortScratch {
  size_t keys[2], perm[2], flag, scan, temp, temp_bytes, end;
};

// Lays the sort scratch of N rows out from byte offset `at`.  Nonzero when the sort's workspace query fails.
static int sid_sort_scratch(int64_t N, int levels, size_t at, SidSortScratch& s) {
  size_t sort_bytes = 0, scan_bytes = 0;
  const int n = (int)N > 0 ? (int)N : 1;
  if (cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                      (const int*)nullptr, (int*)nullptr, n, 0, 64) != cudaSuccess ||
      cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, n) != cudaSuccess) {
    cudaGetLastError();
    return 1;
  }
  s.temp_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
  for (int i = 0; i < 2; ++i) {
    s.keys[i] = at;
    at += sid_align256((size_t)N * sizeof(unsigned long long));
  }
  for (int i = 0; i < 2; ++i) {
    s.perm[i] = at;
    at += sid_align256((size_t)N * sizeof(int));
  }
  s.flag = at;
  at += sid_align256((size_t)levels * N * sizeof(int));
  s.scan = at;
  at += sid_align256((size_t)levels * N * sizeof(int));
  s.temp = at;
  s.end = at + sid_align256(s.temp_bytes);
  return 0;
}

// The trie's header and workspace bytes: arithmetic only, no device.  Nonzero outside the trie's limits.
static int sid_trie_layout(int64_t N, int C, int K, SidTrieHeader& h, size_t& bytes) {
  if (N < 0 || N >= 0x7fffffffll || C <= 0 || C > 8 || K <= 0 || K > 65536) return 1;
  h = SidTrieHeader{};
  h.C = C;
  h.K = K;
  h.N = N;
  h.n[0] = 1;
  size_t at = sid_align256(sizeof(SidTrieHeader));
  for (int l = 0; l < C; ++l) {
    h.child[l] = at;
    at += sid_align256(((l == 0 ? 1 : (size_t)N) + 1) * sizeof(int));
  }
  for (int l = 1; l <= C; ++l) {
    h.code[l] = at;
    at += sid_align256((size_t)N * sizeof(unsigned short));
  }
  bytes = at;
  return 0;
}

extern "C" size_t rqb200_sid_trie_workspace_bytes(int64_t N, int C, int K) {
  SidTrieHeader h;
  size_t bytes;
  return sid_trie_layout(N, C, K, h, bytes) ? 0 : bytes;
}

extern "C" size_t rqb200_sid_trie_scratch_bytes(int64_t N, int C, int K) {
  SidTrieHeader h;
  size_t bytes;
  SidSortScratch s;
  return (sid_trie_layout(N, C, K, h, bytes) || sid_sort_scratch(N, C, 0, s)) ? 0 : s.end;
}

// number of leading ids of a row inside [0, K)
__device__ __forceinline__ int sid_row_depth(const int64_t* row, int C, int K) {
  int d = 0;
  while (d < C && row[d] >= 0 && row[d] < K) ++d;
  return d;
}

__global__ void sid_trie_header_kernel(SidTrieHeader h, unsigned char* ws) {
  *reinterpret_cast<SidTrieHeader*>(ws) = h;
  int* child0 = reinterpret_cast<int*>(ws + h.child[0]);
  child0[0] = 0;
  child0[1] = 0;                                            // n[1]; the fill pass writes it when N > 0
}

__global__ void sid_trie_iota_kernel(int* perm, int N) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) perm[i] = i;
}

// ids c0 .. c1 - 1 of a row, `width` bits each, the first id most significant; ids at or after position d are K
__device__ __forceinline__ unsigned long long sid_pack_cols(const int64_t* row, int d, int c0, int c1, int width, int K) {
  unsigned long long key = 0;
  for (int c = c0; c < c1; ++c) key = (key << width) | (unsigned long long)(c < d ? row[c] : K);
  return key;
}

// keys[i] = ids c0 .. c1 - 1 of row perm[i] packed, ids at or after the row's first id outside [0, K) K
__global__ void sid_trie_key_kernel(const int64_t* __restrict__ ids, int N, int C, int K, const int* __restrict__ perm, int c0, int c1,
                                    int width, unsigned long long* __restrict__ keys) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
    const int64_t* row = ids + (int64_t)perm[i] * C;
    keys[i] = sid_pack_cols(row, sid_row_depth(row, C, K), c0, c1, width, K);
  }
}

// the item table's sort key: as sid_trie_key_kernel, but a row holding any id outside [0, K) is all K (it sorts last)
__global__ void sid_items_key_kernel(const int64_t* __restrict__ ids, int N, int C, int K, const int* __restrict__ perm, int c0, int c1,
                                     int width, unsigned long long* __restrict__ keys) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
    const int64_t* row = ids + (int64_t)perm[i] * C;
    keys[i] = sid_pack_cols(row, sid_row_depth(row, C, K) == C ? C : 0, c0, c1, width, K);
  }
}

// Stable LSD radix sort of the N rows on their packed tuple, least significant column group first (CUB, on the stream), in the
// sort scratch s at `scratch`.  `sorted` ends pointing at the sorted row ids; with `whole` rows that hold an id outside [0, K)
// sort last, else the trie's order.
static int sid_sort_rows(const int64_t* ids, int n, int C, int K, bool whole, unsigned char* scratch, const SidSortScratch& s,
                         int grid, cudaStream_t st, int*& sorted) {
  unsigned long long* keys[2] = {reinterpret_cast<unsigned long long*>(scratch + s.keys[0]),
                                 reinterpret_cast<unsigned long long*>(scratch + s.keys[1])};
  int* perm[2] = {reinterpret_cast<int*>(scratch + s.perm[0]), reinterpret_cast<int*>(scratch + s.perm[1])};
  const int width = sid_id_bits(K), cols = 64 / width;
  sid_trie_iota_kernel<<<grid, 256, 0, st>>>(perm[0], n);
  RQB_LAUNCH_CHECK();
  const int groups = (C + cols - 1) / cols;
  for (int g = groups - 1; g >= 0; --g) {                   // least significant column group first; each sort is stable
    const int c0 = g * cols, c1 = min(C, c0 + cols);
    if (whole) sid_items_key_kernel<<<grid, 256, 0, st>>>(ids, n, C, K, perm[0], c0, c1, width, keys[0]);
    else sid_trie_key_kernel<<<grid, 256, 0, st>>>(ids, n, C, K, perm[0], c0, c1, width, keys[0]);
    RQB_LAUNCH_CHECK();
    size_t tb = s.temp_bytes;
    RQB_CUDA(cub::DeviceRadixSort::SortPairs(scratch + s.temp, tb, keys[0], keys[1], perm[0], perm[1], n, 0, width * (c1 - c0), st));
    std::swap(perm[0], perm[1]);
  }
  sorted = perm[0];
  return RQB_OK;
}

// flag[l - 1][r] = sorted row r starts a node of level l: l is within its valid length and beyond its common prefix with row r - 1
__global__ void sid_trie_flag_kernel(const int64_t* __restrict__ ids, int N, int C, int K, const int* __restrict__ perm,
                                     int* __restrict__ flag) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < N; r += gridDim.x * blockDim.x) {
    const int64_t* row = ids + (int64_t)perm[r] * C;
    const int d = sid_row_depth(row, C, K);
    int lcp = 0;
    if (r > 0) {
      const int64_t* prev = ids + (int64_t)perm[r - 1] * C;
      const int m = min(d, sid_row_depth(prev, C, K));
      while (lcp < m && prev[lcp] == row[lcp]) ++lcp;
    }
    for (int l = 1; l <= C; ++l) flag[(int64_t)(l - 1) * N + r] = (l > lcp && l <= d) ? 1 : 0;
  }
}

// scan[l - 1][r] = nodes of level l started by sorted rows 0..r.  Row r writes the code of every node it starts and, for every
// node p of level l - 1 it starts (the root: row 0), child_{l-1}[p] = the nodes of level l started before row r; the last row
// closes every child array and stores the node counts.
__global__ void sid_trie_fill_kernel(const int64_t* __restrict__ ids, int N, int C, const int* __restrict__ perm,
                                     const int* __restrict__ flag, const int* __restrict__ scan, unsigned char* ws) {
  SidTrieHeader* hdr = reinterpret_cast<SidTrieHeader*>(ws);
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < N; r += gridDim.x * blockDim.x) {
    const int64_t* row = ids + (int64_t)perm[r] * C;
    for (int l = 1; l <= C; ++l) {
      const int f = flag[(int64_t)(l - 1) * N + r], s = scan[(int64_t)(l - 1) * N + r];
      if (f) reinterpret_cast<unsigned short*>(ws + hdr->code[l])[s - 1] = (unsigned short)row[l - 1];
      const bool starts_parent = l == 1 ? r == 0 : flag[(int64_t)(l - 2) * N + r] != 0;
      if (starts_parent) {
        const int p = l == 1 ? 0 : scan[(int64_t)(l - 2) * N + r] - 1;
        reinterpret_cast<int*>(ws + hdr->child[l - 1])[p] = s - f;
      }
    }
    if (r == N - 1) {
      int np = 1;
      for (int l = 1; l <= C; ++l) {
        const int nl = scan[(int64_t)(l - 1) * N + r];
        reinterpret_cast<int*>(ws + hdr->child[l - 1])[np] = nl;
        hdr->n[l] = nl;
        np = nl;
      }
    }
  }
}

extern "C" int rqb200_sid_trie_build(const int64_t* cached_ids, int64_t N, int C, int K, void* workspace, size_t ws_bytes,
                                     void* scratch, size_t scratch_bytes, void* stream) {
  RQB_CHECK_ARG(N >= 0 && C > 0 && C <= 8 && K > 0 && workspace, "sid_trie_build: bad argument");
  SidTrieHeader h;
  size_t bytes;
  if (sid_trie_layout(N, C, K, h, bytes)) {
    rqb_set_error("sid_trie_build: need N < 2^31 - 1 and K <= 65536 (N = %lld, K = %d)", (long long)N, K);
    return RQB_ERR_UNSUPPORTED;
  }
  SidSortScratch s;
  if (sid_sort_scratch(N, C, 0, s)) {
    rqb_set_error("sid_trie_build: the sort's workspace query failed (no CUDA device?)");
    return RQB_ERR_CUDA;
  }
  if (ws_bytes < bytes) {
    rqb_set_error("sid_trie_build: workspace too small");
    return RQB_ERR_WORKSPACE;
  }
  if (scratch_bytes < s.end) {
    rqb_set_error("sid_trie_build: scratch too small");
    return RQB_ERR_WORKSPACE;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  sid_trie_header_kernel<<<1, 1, 0, st>>>(h, ws);
  RQB_LAUNCH_CHECK();
  if (N == 0) return RQB_OK;
  RQB_CHECK_ARG(cached_ids && scratch, "sid_trie_build: null pointer");
  const int n = (int)N;
  int grid = (n + 255) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  unsigned char* sc = reinterpret_cast<unsigned char*>(scratch);
  int* flag = reinterpret_cast<int*>(sc + s.flag);
  int* scan = reinterpret_cast<int*>(sc + s.scan);
  int* sorted = nullptr;
  const int rc = sid_sort_rows(cached_ids, n, C, K, false, sc, s, grid, st, sorted);
  if (rc != RQB_OK) return rc;
  sid_trie_flag_kernel<<<grid, 256, 0, st>>>(cached_ids, n, C, K, sorted, flag);
  RQB_LAUNCH_CHECK();
  for (int l = 0; l < C; ++l) {
    size_t temp_bytes = s.temp_bytes;
    RQB_CUDA(cub::DeviceScan::InclusiveSum(sc + s.temp, temp_bytes, flag + (int64_t)l * n, scan + (int64_t)l * n, n, st));
  }
  sid_trie_fill_kernel<<<grid, 256, 0, st>>>(cached_ids, n, C, sorted, flag, scan, ws);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// The trie's level arrays as plain device arrays, for the exact ranking of modules/model.py (rank_sem_ids), which decodes one
// row per trie node.  rqb200_sid_trie_counts copies the node counts n[0..C] to a device array (the caller reads them once per
// index); rqb200_sid_trie_level writes, for level l (1..C), each node's code, its parent in level l - 1 (from the parent's
// child range) and, for l < C, its child range in level l + 1 (child[n_l + 1]).
__global__ void sid_trie_counts_kernel(const unsigned char* __restrict__ ws, int* __restrict__ counts) {
  const SidTrieHeader* hdr = reinterpret_cast<const SidTrieHeader*>(ws);
  for (int l = threadIdx.x; l <= hdr->C; l += blockDim.x) counts[l] = hdr->n[l];
}

__global__ void sid_trie_level_kernel(const unsigned char* __restrict__ ws, int l, int n_l, int n_prev, int* __restrict__ code,
                                      int* __restrict__ parent, int* __restrict__ child) {
  const SidTrieHeader* hdr = reinterpret_cast<const SidTrieHeader*>(ws);
  const unsigned short* c = reinterpret_cast<const unsigned short*>(ws + hdr->code[l]);
  const int* up = reinterpret_cast<const int*>(ws + hdr->child[l - 1]);
  const int* down = l < hdr->C ? reinterpret_cast<const int*>(ws + hdr->child[l]) : nullptr;
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= n_l; i += stride) {
    if (i < n_l) code[i] = c[i];
    if (child) child[i] = down ? down[i] : 0;
  }
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n_prev; p += stride)
    for (int j = up[p]; j < up[p + 1]; ++j) parent[j] = p;
}

extern "C" int rqb200_sid_trie_counts(const void* workspace, int* counts, void* stream) {
  RQB_CHECK_ARG(workspace && counts, "sid_trie_counts: null pointer");
  sid_trie_counts_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const unsigned char*>(workspace),
                                                                             counts);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_sid_trie_level(const void* workspace, int C, int l, int n_l, int n_prev, int* code, int* parent, int* child,
                                     void* stream) {
  RQB_CHECK_ARG(C > 0 && C <= 8 && l >= 1 && l <= C && n_l >= 0 && n_prev >= 0,
                "sid_trie_level: bad argument (C = %d, l = %d, n_l = %d, n_prev = %d)", C, l, n_l, n_prev);
  RQB_CHECK_ARG(workspace && code && parent && (l == C || child), "sid_trie_level: null pointer");
  int grid = (n_l + 256) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  sid_trie_level_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const unsigned char*>(workspace), l, n_l, n_prev, code, parent, l < C ? child : nullptr);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Lookups in the trie.  A search kernel tests "the beam's prefix extended by code tok is a corpus prefix" through
//   parent(ids, h, K)    the walk from the root along the beam's ids [0, h): the range of its children at level h + 1;
//   has(parent, tok, K)  one binary search among those children;
//   prefix(ids, l, K)    ids[0, l) is a corpus prefix (the check kernel);
//   sid_child_mask       the children's codes as a K-bit mask in shared memory, so that a candidate's test is one bit test
//                        (sample_select and beam_topk, which hold one beam per warp at a time or every beam of a row).
// A SidTrie object serves one prefix length: `level` = h + 1 in the search kernels, l in the check kernel.
struct SidTrie {                                            // the whole trie workspace
  const unsigned char* ws;
  int level;
  struct Parent { int lo, hi; };                            // the beam's children: nodes [lo, hi) of `level` (empty: not a prefix)
  __device__ __forceinline__ const SidTrieHeader* hdr() const { return reinterpret_cast<const SidTrieHeader*>(ws); }
  __device__ __forceinline__ const int* child(int l) const { return reinterpret_cast<const int*>(ws + __ldg(&hdr()->child[l])); }
  __device__ __forceinline__ const unsigned short* code(int l) const {
    return reinterpret_cast<const unsigned short*>(ws + __ldg(&hdr()->code[l]));
  }
  // position of code v among the sorted codes c[lo, hi), or -1
  __device__ __forceinline__ static int find(const unsigned short* c, int lo, int hi, int64_t v) {
    int a = lo, b = hi;
    while (a < b) {
      const int mid = (a + b) >> 1;
      if ((int64_t)__ldg(c + mid) < v) a = mid + 1;
      else b = mid;
    }
    return (a < hi && (int64_t)__ldg(c + a) == v) ? a : -1;
  }
  __device__ __forceinline__ Parent parent(const int64_t* ids, int h, int K) const {
    const int* c0 = child(0);
    int lo = __ldg(c0), hi = __ldg(c0 + 1);
    for (int j = 0; j < h; ++j) {
      const int64_t v = ids[j];
      const int n = (v >= 0 && v < K) ? find(code(j + 1), lo, hi, v) : -1;
      if (n < 0) return {0, 0};
      const int* c = child(j + 1);
      lo = __ldg(c + n);
      hi = __ldg(c + n + 1);
    }
    return {lo, hi};
  }
  __device__ __forceinline__ bool has(const Parent& p, int64_t tok, int K) const {
    return tok >= 0 && tok < K && find(code(level), p.lo, p.hi, tok) >= 0;
  }
  __device__ __forceinline__ bool prefix(const int64_t* ids, int l, int K) const { return has(parent(ids, l - 1, K), ids[l - 1], K); }
};

// One warp: mask[0, ceil(K / 32)) = bit c set for every child code c of the beam ids[0, h) (none when the beam is not a corpus
// prefix).  The warp is synchronised on return.
__device__ __forceinline__ void sid_child_mask(const SidTrie& trie, const int64_t* ids, int h, int K, unsigned int* mask, int lane) {
  const SidTrie::Parent par = trie.parent(ids, h, K);
  const unsigned short* code = trie.code(h + 1);
  for (int i = lane; i < (K + 31) >> 5; i += 32) mask[i] = 0;
  __syncwarp();
  for (int i = par.lo + lane; i < par.hi; i += 32) {
    const int c = __ldg(code + i);
    atomicOr(&mask[c >> 5], 1u << (c & 31));
  }
  __syncwarp();
}

__device__ __forceinline__ bool sid_mask_has(const unsigned int* mask, int c) { return (mask[c >> 5] >> (c & 31)) & 1u; }

// One warp, after sid_child_mask: clears the bits of the beam's children that are blocked for history b (SidExcl), the keys
// [key(ids[0, h)) K, key(ids[0, h)) K + K) of level h + 1's blocked list.  Nothing to do without an exclusion.  The warp is
// synchronised on return.
__device__ __forceinline__ void sid_mask_unblock(const SidExcl& ex, int64_t b, const int64_t* ids, int h, int K, unsigned int* mask,
                                                 int lane) {
  if (!ex.on()) return;
  long long key = 0;
  for (int j = 0; j < h; ++j) {
    const int64_t v = ids[j];
    key = key * K + (v < 0 ? 0 : v >= K ? K - 1 : v);       // a beam holding such an id is no corpus prefix: its mask is empty
  }
  const long long lo = key * K, hi = lo + K;
  const long long* list = ex.keys_of(b, h + 1);
  const int n = ex.nkeys(b, h + 1);
  for (int i = sid_lower_bound(list, n, lo) + lane; i < n && __ldg(list + i) < hi; i += 32) {
    const int c = (int)(__ldg(list + i) - lo);
    atomicAnd(&mask[c >> 5], ~(1u << (c & 31)));
  }
  __syncwarp();
}

// One warp, with an allow-list (SidExcl::include): mask = bit c set for every child code c of the beam ids[0, h) that is valid
// for history b, the keys [key(ids[0, h)) K, key(ids[0, h)) K + K) of level h + 1's allowed list (two binary searches).  The
// allowed keys are corpus prefixes, so the trie is not read.  The warp is synchronised on return.
__device__ __forceinline__ void sid_allowed_mask(const SidExcl& in, int64_t b, const int64_t* ids, int h, int K, unsigned int* mask,
                                                 int lane) {
  for (int i = lane; i < (K + 31) >> 5; i += 32) mask[i] = 0;
  long long key = 0;
  bool ok = true;                                           // a beam holding an id outside [0, K) has no valid child
  for (int j = 0; j < h; ++j) {
    const int64_t v = ids[j];
    ok &= v >= 0 && v < K;
    key = key * K + (ok ? v : 0);
  }
  __syncwarp();
  if (ok) {
    const long long lo = key * K;
    const long long* list = in.keys_of(b, h + 1);
    const int n = in.nkeys(b, h + 1);
    const int end = sid_lower_bound(list, n, lo + K);
    for (int i = sid_lower_bound(list, n, lo) + lane; i < end; i += 32) {
      const int c = (int)(__ldg(list + i) - lo);
      atomicOr(&mask[c >> 5], 1u << (c & 31));
    }
  }
  __syncwarp();
}

// One warp: the K-bit mask of the beam's valid children under the consumer's filter mode (SidFilterMode): the trie's children,
// less the blocked ones with an exclusion, or the allowed ones with an inclusion.  The warp is synchronised on return.
template <int FILTER>
__device__ __forceinline__ void sid_beam_mask(const SidTrie& trie, const SidExcl& f, int64_t b, const int64_t* ids, int h, int K,
                                              unsigned int* mask, int lane) {
  if (FILTER == SID_FILTER_INCLUDE) {
    sid_allowed_mask(f, b, ids, h, K, mask, lane);
    return;
  }
  sid_child_mask(trie, ids, h, K, mask, lane);
  if (FILTER == SID_FILTER_EXCLUDE) sid_mask_unblock(f, b, ids, h, K, mask, lane);
}

// the filter mode of a filter argument (count null: none)
__host__ __forceinline__ int sid_filter_mode(const SidExcl& f) {
  return !f.count ? SID_FILTER_NONE : f.include ? SID_FILTER_INCLUDE : SID_FILTER_EXCLUDE;
}

// valid[p] = any corpus row whose first l ids equal prefix[p, :l]      (model.py:175-181)
__global__ void sid_prefix_check_kernel(const int64_t* __restrict__ prefix, int64_t stride, int64_t P, int l, int K, SidTrie trie,
                                        unsigned char* __restrict__ valid) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (int64_t)gridDim.x * blockDim.x)
    valid[p] = trie.prefix(prefix + p * stride, l, K) ? 1 : 0;
}

extern "C" int rqb200_sid_trie_check(const int64_t* prefix, int64_t row_stride, int64_t P, int l, int C, int K, const void* workspace,
                                     unsigned char* valid, void* stream) {
  RQB_CHECK_ARG(P >= 0 && l > 0 && l <= C && C <= 8 && K > 0 && row_stride >= l, "sid_trie_check: bad argument (l=%d C=%d)", l, C);
  if (P == 0) return RQB_OK;
  RQB_CHECK_ARG(prefix && workspace && valid, "sid_trie_check: null pointer");
  int grid = (int)((P + 255) / 256);
  if (grid > 132 * 16) grid = 132 * 16;
  sid_prefix_check_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      prefix, row_stride, P, l, K, SidTrie{reinterpret_cast<const unsigned char*>(workspace), l}, valid);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// One selection step of the constrained beam search (modules/model.py:340-376) in one launch: for every batch row the
// kp x nc candidate extensions (kp live beams, nc sampled tokens each) are scored  log p(token) + log p(parent beam),  the
// extensions whose id prefix does not occur in the corpus get -inf (the trie above: the reference's repeat_interleave + cat +
// O(P N) compare + masked_fill), and the k best are taken in descending score order (the reference sorts all kp nc scores and
// keeps k), with their ids gathered into the new beams and the parent beam's global index returned for the key/value-cache
// reorder.  Ties: lowest flat candidate index first (torch.sort is not stable: any order is legal).
// One warp per batch row; kp * nc <= 1024, k <= 32.  Each warp first resolves its row's kp beams in the trie (shared memory),
// then tests each candidate with one binary search among its beam's children: a K-bit mask per beam would not fit for
// 1024 beams.
#define SID_BEAM_MAX_E 1024

// Score of one candidate extension: lp (token log-probability + parent beam log-probability), or -inf when the prefix
// parent ids + tok is not in the corpus (!valid, model.py:356,366) or lp is NaN (NaN ranks last here).
__device__ __forceinline__ float sid_extension_score(bool valid, float lp) { return (!valid || lp != lp) ? -INFINITY : lp; }

// One warp keeps the k best of batch row b's E = kp * nc candidate scores sc[] in descending order: k rounds of a warp
// arg-max over the candidates not yet taken (tk[], cleared by the caller).  tok[e] is candidate e's token (e = beam * nc + j).
// Writes the new beams, their scores and the parent beam's global index b * kp + beam.
__device__ __forceinline__ void sid_keep_best(const float* sc, unsigned char* tk, const int64_t* tok, int E, int nc, int b, int kp,
                                              int h, int k, const int64_t* __restrict__ generated, int64_t* __restrict__ out_generated,
                                              float* __restrict__ out_log_probas, int64_t* __restrict__ out_parent, int lane) {
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
      out_generated[((int64_t)b * k + r) * (h + 1) + h] = tok[bi];
    }
    for (int j = lane; j < h; j += 32)
      out_generated[((int64_t)b * k + r) * (h + 1) + j] = generated[((int64_t)b * kp + beam) * h + j];
    __syncwarp();
  }
}

__global__ void __launch_bounds__(128) sid_beam_select_kernel(
    const int64_t* __restrict__ samples, const float* __restrict__ samp_log_p, const int64_t* __restrict__ generated,
    const float* __restrict__ log_probas, int B, int kp, int nc, int h, int k, int K, SidTrie trie,
    int64_t* __restrict__ out_generated, float* __restrict__ out_log_probas, int64_t* __restrict__ out_parent) {
  extern __shared__ __align__(16) unsigned char sid_smem[];
  __shared__ float s_score[4][SID_BEAM_MAX_E];
  __shared__ unsigned char s_taken[4][SID_BEAM_MAX_E];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * 4 + w;
  if (b >= B) return;
  const int E = kp * nc;
  float* sc = s_score[w];
  unsigned char* tk = s_taken[w];
  SidTrie::Parent* s_par = reinterpret_cast<SidTrie::Parent*>(sid_smem) + w * kp;   // [4][kp]: the row's beams, resolved once
  for (int beam = lane; beam < kp; beam += 32) s_par[beam] = trie.parent(generated + ((int64_t)b * kp + beam) * h, h, K);
  __syncwarp();
  for (int e = lane; e < E; e += 32) {
    const int beam = e / nc;
    const int64_t row = (int64_t)b * kp + beam;
    const float s = samp_log_p[row * nc + (e - beam * nc)] + (log_probas ? log_probas[row] : 0.f);
    sc[e] = sid_extension_score(trie.has(s_par[beam], samples[row * nc + (e - beam * nc)], K), s);
    tk[e] = 0;
  }
  __syncwarp();
  sid_keep_best(sc, tk, samples + (int64_t)b * kp * nc, E, nc, b, kp, h, k, generated, out_generated, out_log_probas, out_parent, lane);
}

extern "C" int rqb200_sid_trie_beam_select(const int64_t* samples, const float* samp_log_p, const int64_t* generated,
                                           const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K,
                                           const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                           int64_t* out_parent, void* stream) {
  RQB_CHECK_ARG(B >= 0 && kp > 0 && nc > 0 && h >= 0 && h < C && C <= 8 && k > 0 && K > 0, "sid_trie_beam_select: bad argument");
  if (kp * nc > SID_BEAM_MAX_E || k > 32) {
    rqb_set_error("sid_trie_beam_select: kp * nc = %d (max %d), k = %d (max 32)", kp * nc, SID_BEAM_MAX_E, k);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(samples && samp_log_p && prefix_workspace && out_generated && out_log_probas && out_parent && (h == 0 || generated),
                "sid_trie_beam_select: null pointer");
  const size_t smem = 4 * (size_t)kp * sizeof(SidTrie::Parent);
  RQB_CUDA(cudaFuncSetAttribute(sid_beam_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  sid_beam_select_kernel<<<(B + 3) / 4, 128, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      samples, samp_log_p, generated, log_probas, B, kp, nc, h, k, K,
      SidTrie{reinterpret_cast<const unsigned char*>(prefix_workspace), h + 1}, out_generated, out_log_probas, out_parent);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// The sampling step of the beam search fused with the selection step above (modules/model.py:344-388 after the softmax).
// torch.multinomial(p, n) without replacement is topk(p / q, n) with q = empty_like(p).exponential_(1) drawn from the same
// generator; given that q, this kernel reproduces its samples bit for bit: ratio = p / q as an IEEE fp32 division (at::div),
// the n largest ratios in torch.topk's order (descending; NaN above +inf and -0 below +0, as its radix selection ranks them;
// equal ratios by ascending index, as its gather and stable sort leave them), samp_log_p = logf(p[sample]).  The candidates
// then go through sid_extension_score / sid_keep_best exactly as in rqb200_sid_trie_beam_select.
// One CTA per batch row; warp w samples beams w, w + W, ... (W = min(kp, 16)) from its own shared-memory copy of the row's
// ratio keys, expands each beam's children into its own K-bit mask (sid_child_mask) and tests its candidates against it; warp 0
// then selects from the kp * nc candidates.  Nothing is ordered by atomics: the results are deterministic.
#define SID_SAMPLE_MAX_WARPS 16
#define SID_SAMPLE_MAX_K 2048

// Order-preserving image of an fp32 value in the order torch.topk's radix selection uses: NaN largest, -0 below +0.
__device__ __forceinline__ unsigned int sid_topk_key(float v) {
  const unsigned int x = __float_as_uint(v);
  return v == v ? x ^ ((x & 0x80000000u) ? 0xffffffffu : 0x80000000u) : 0xffffffffu;
}

// One warp: the indices of the n largest of key[0..K) into out[0..n), descending, equal keys by ascending index.  Radix
// selection of the n-th largest key T (four 8-bit digits, shared histogram hist[256]), compaction of every key above T and of
// the lowest-index keys equal to T (index order, sel_key / sel_idx [n]), then each kept key's rank among the kept ones.
__device__ void sid_warp_top_n(const unsigned int* key, int K, int n, int* hist, unsigned int* sel_key, int* sel_idx, int64_t* out,
                               int lane) {
  const unsigned int lt = (1u << lane) - 1u;
  unsigned int prefix = 0, pmask = 0;
  int want = n;                                             // entries still needed among those matching the decided digits
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = lane; i < 256; i += 32) hist[i] = 0;
    __syncwarp();
    for (int base = 0; base < K; base += 32) {
      const int i = base + lane;
      const unsigned int v = i < K ? key[i] : 0u;
      const int d = (i < K && (v & pmask) == prefix) ? (int)((v >> shift) & 255u) : 256;
      const unsigned int same = __match_any_sync(0xffffffffu, d);
      if (d < 256 && (same & lt) == 0) atomicAdd(&hist[d], __popc(same));   // one add per distinct digit of the 32 keys
    }
    __syncwarp();
    int c[8], s = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { c[j] = hist[lane * 8 + j]; s += c[j]; }
    int suf = s;                                            // entries in bins >= lane * 8
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_down_sync(0xffffffffu, suf, o);
      if (lane + o < 32) suf += t;
    }
    const int owner = 31 - __clz(__ballot_sync(0xffffffffu, suf >= want));   // the lane holding the n-th largest digit
    int digit = 0, above = 0;
    if (lane == owner) {
      int acc = suf - s;
      for (int j = 7; j >= 0; --j) {
        if (acc + c[j] >= want) { digit = lane * 8 + j; above = acc; break; }
        acc += c[j];
      }
    }
    digit = __shfl_sync(0xffffffffu, digit, owner);
    above = __shfl_sync(0xffffffffu, above, owner);
    want -= above;
    prefix |= (unsigned int)digit << shift;
    pmask |= 255u << shift;
    __syncwarp();
  }
  int kept = 0, eq_seen = 0;                                // keys above T: n - want of them; keys equal to T: the first `want`
  for (int base = 0; base < K; base += 32) {
    const int i = base + lane;
    const unsigned int v = i < K ? key[i] : 0u;
    const bool eq = i < K && v == prefix;
    const unsigned int beq = __ballot_sync(0xffffffffu, eq);
    const bool take = (i < K && v > prefix) || (eq && eq_seen + __popc(beq & lt) < want);
    const unsigned int bt = __ballot_sync(0xffffffffu, take);
    if (take) {
      sel_key[kept + __popc(bt & lt)] = v;
      sel_idx[kept + __popc(bt & lt)] = i;
    }
    kept += __popc(bt);
    eq_seen += __popc(beq);
  }
  __syncwarp();
  for (int p = lane; p < n; p += 32) {
    const unsigned int v = sel_key[p];
    int r = 0;
    for (int q = 0; q < n; ++q) {
      const unsigned int u = sel_key[q];
      r += (u > v) || (u == v && q < p);
    }
    out[r] = sel_idx[p];
  }
  __syncwarp();
}

// ---------------------------------------------------------------------------------------------------------------------
// The warped draw: a sampling mode of sid_sample_select_kernel / sid_sample_select_wide_kernel that draws from the head's
// logits at a temperature T and within a top-p nucleus.  Per beam row x[0, K), one warp:
//   m = max x,  lse = m + logf(sum expf(x - m))             (sid_beam_topk_kernel's statement and order)
//   p_T[c] = expf((x[c] - m) / T) / S,  S = sum_c expf((x[c] - m) / T)   (fp32, lane-strided sums, then a butterfly)
//   N = {c : p_T[c] >= t}, t the largest p_T with mass(p_T >= t) >= top_p * mass(all)   (ties at t all in; top_p = 1: all)
// where mass sums fx(p_T) = floor(p_T * 2^40) as 64-bit integers, so it is independent of any order.  The keys of the codes
// of N with p_T > 0 (N+) are sid_topk_key(p_T / q), those of every other code 0 (below every ratio's key: sid_warp_top_n
// draws them last, as -inf fillers).  A row with a NaN or +inf, or all -inf, has every key 0 and is reported bad.
#define SID_FX_ONE 1099511627776.f                          // 2^40: fixed-point unit of the nucleus masses

__device__ __forceinline__ unsigned long long sid_fx(float p) { return __float2ull_rz(p * SID_FX_ONE); }

// One warp: the bits of t over the p_T bits key[0, K) (non-negative floats: their bits order as their values), given
// 0 < target <= the total mass.  Radix selection on 7-bit digits (bits 31..4 in four passes, then 3..0) of integer mass
// histograms hist[128]: each pass keeps the largest digit whose bin, with the larger bins and the mass above, reaches target.
// The chosen bin always holds mass, so t is some code's p_T.
__device__ __forceinline__ unsigned int sid_nucleus_threshold(const unsigned int* key, int K, unsigned long long target, unsigned long long* hist,
                                              int lane) {
  unsigned int prefix = 0, pmask = 0;
  unsigned long long above = 0;                             // mass of the codes above the decided digits
  for (int pass = 0; pass < 5; ++pass) {
    const int shift = pass < 4 ? 25 - 7 * pass : 0;
    const unsigned int dmask = pass < 4 ? 127u : 15u;
    for (int i = lane; i < 128; i += 32) hist[i] = 0;
    __syncwarp();
    for (int c = lane; c < K; c += 32) {
      const unsigned int v = key[c];
      if ((v & pmask) != prefix) continue;
      const unsigned long long f = sid_fx(__uint_as_float(v));
      if (f) atomicAdd(&hist[(v >> shift) & dmask], f);
    }
    __syncwarp();
    unsigned long long s = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) s += hist[lane * 4 + j];
    unsigned long long suf = s;                             // mass in bins >= lane * 4
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long t = __shfl_down_sync(0xffffffffu, suf, o);
      if (lane + o < 32) suf += t;
    }
    const int owner = 31 - __clz(__ballot_sync(0xffffffffu, above + suf >= target));
    int digit = 0;
    unsigned long long acc = 0;
    if (lane == owner) {
      acc = above + suf - s;
      for (int j = 3; j >= 0; --j) {
        const unsigned long long c = hist[lane * 4 + j];
        if (acc + c >= target) { digit = lane * 4 + j; break; }
        acc += c;
      }
    }
    digit = __shfl_sync(0xffffffffu, digit, owner);
    above = __shfl_sync(0xffffffffu, acc, owner);
    prefix |= (unsigned int)digit << shift;
    pmask |= dmask << shift;
    __syncwarp();
  }
  return prefix;
}

struct SidWarpedRow {
  float lse;
  bool bad;
};

// One warp, beam row x / noise q: key[0, K) = the warped draw's keys (above), hist = 128 64-bit bins of scratch (8-byte
// aligned).  Returns the row's lse and whether it is bad.  The warp is synchronised on return.
__device__ __forceinline__ SidWarpedRow sid_warped_keys(const float* __restrict__ x, const float* __restrict__ q, int K, float temp, double top_p,
                                        unsigned int* key, unsigned long long* hist, int lane) {
  float m = -INFINITY;
  bool odd = false;
  for (int c = lane; c < K; c += 32) {
    const float v = x[c];
    m = fmaxf(m, v);
    odd |= v != v || v == INFINITY;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  odd = __any_sync(0xffffffffu, odd);
  const bool bad = odd || m == -INFINITY;
  float sum = 0.f, st = 0.f;
  for (int c = lane; c < K; c += 32) {
    const float v = x[c];
    sum += expf(v - m);
    const float e = expf(__fdiv_rn(__fsub_rn(v, m), temp));
    st = __fadd_rn(st, e);
    key[c] = bad ? 0u : __float_as_uint(e);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);            // every lane ends with the same bits
    st = __fadd_rn(st, __shfl_xor_sync(0xffffffffu, st, o));
  }
  const float lse = m + logf(sum);
  __syncwarp();
  if (bad) return {lse, true};
  unsigned long long total = 0;                             // S >= 1: the maximum's term is expf(0) = 1
  for (int c = lane; c < K; c += 32) {
    const float p = __fdiv_rn(__uint_as_float(key[c]), st);
    key[c] = __float_as_uint(p);
    total += sid_fx(p);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
  __syncwarp();
  unsigned int t = 0;
  if (top_p < 1.0) {
    const unsigned long long target = (unsigned long long)ceil(top_p * (double)total);
    t = sid_nucleus_threshold(key, K, target < 1 ? 1 : target, hist, lane);
  }
  for (int c = lane; c < K; c += 32) {
    const unsigned int v = key[c];
    key[c] = (v >= t && v != 0u) ? sid_topk_key(__fdiv_rn(__uint_as_float(v), q[c])) : 0u;
  }
  __syncwarp();
  return {lse, false};
}

template <bool WARP>
static size_t sid_sample_smem(int kp, int nc, int K) {
  const int W = kp < SID_SAMPLE_MAX_WARPS ? kp : SID_SAMPLE_MAX_WARPS;
  const size_t E = (size_t)kp * nc;
  return E * (sizeof(int64_t) + sizeof(float) + 1) + (size_t)W * (K + 256 + 2 * nc + (K + 31) / 32) * 4 + (WARP ? 4 : 0);
}

// ---------------------------------------------------------------------------------------------------------------------
// The per-prefix cap (CAP mode of sid_beam_topk_kernel and sid_sample_select_kernel): at a level h >= len, at most m of a
// history's kept beams with a finite score share their first len ids.  A candidate's group is its parent beam's len-prefix,
// named by the lowest beam of the row with an equal prefix.  The kept set is the greedy walk down the uncapped order (score
// descending, lowest flat index first) that skips a candidate whose group already holds m: it keeps each group's m best
// candidates and drops the rest to -inf, where they rank among the -inf fillers by flat index as every filler does.  A group
// holding fewer than m finite candidates loses none; -inf candidates are unchanged either way.
struct SidCap {
  int len;                                                  // prefix length, 1 <= len <= h
  int m;                                                    // most kept beams per group, 1 <= m < k (m >= k cannot bind)
};

// WARP: the warped draw (above) from the head's logits (`probas` holds them), else the untempered draw from the softmax.
// CAP: the per-prefix cap (SidCap, defined with sid_beam_topk_kernel) on the selection; the draws do not change.
template <int FILTER, bool WARP, bool CAP = false>          // SidFilterMode: the filter's code is compiled only with one
__global__ void __launch_bounds__(SID_SAMPLE_MAX_WARPS * 32, WARP ? 1 : 0) sid_sample_select_kernel(
    const float* __restrict__ probas, int64_t p_stride, const float* __restrict__ noise, int64_t n_stride,
    const int64_t* __restrict__ generated, const float* __restrict__ log_probas, int kp, int nc, int h, int k, int K, SidTrie trie,
    int64_t* __restrict__ out_generated, float* __restrict__ out_log_probas, int64_t* __restrict__ out_parent,
    int64_t* __restrict__ samples, float* __restrict__ samp_log_p, int* __restrict__ reject, SidExcl ex, float temp,
    double top_p, SidCap cap) {
  extern __shared__ __align__(16) unsigned char sid_smem[];
  const int W = blockDim.x >> 5, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x, E = kp * nc, KW = (K + 31) >> 5;
  int64_t* s_tok = reinterpret_cast<int64_t*>(sid_smem);                          // [E] candidate tokens
  float* s_score = reinterpret_cast<float*>(s_tok + E);                          // [E] candidate scores
  unsigned int* s_key = reinterpret_cast<unsigned int*>(s_score + E) + (size_t)w * K;                      // [W][K]
  unsigned int* s_key_end = reinterpret_cast<unsigned int*>(s_score + E) + (size_t)W * K;
  if (WARP) s_key_end += ((E + W * K) & 1);                 // the warped mode's 64-bit histograms: 8-byte aligned
  int* s_hist = reinterpret_cast<int*>(s_key_end) + w * 256;                                               // [W][256]
  unsigned int* s_sk = reinterpret_cast<unsigned int*>(s_hist - w * 256 + W * 256) + w * nc;               // [W][nc]
  int* s_si = reinterpret_cast<int*>(s_sk - w * nc + W * nc) + w * nc;                                     // [W][nc]
  unsigned int* s_mask = reinterpret_cast<unsigned int*>(s_si - w * nc + W * nc) + w * KW;                 // [W][KW]
  unsigned char* s_taken = reinterpret_cast<unsigned char*>(s_mask - w * KW + W * KW);                    // [E]
  for (int beam = w; beam < kp; beam += W) {
    const int64_t row = (int64_t)b * kp + beam;
    const float* p = probas + row * p_stride;
    const float* q = noise + row * n_stride;
    float lse = 0.f;
    if (WARP) {
      const SidWarpedRow wr = sid_warped_keys(p, q, K, temp, top_p, s_key, reinterpret_cast<unsigned long long*>(s_hist), lane);
      lse = wr.lse;
      if (reject && lane == 0 && wr.bad) atomicAdd(reject, 1);
    } else {
      bool bad = false, nonzero = false;
      for (int i = lane; i < K; i += 32) {
        const float pv = p[i];
        bad |= !(pv >= 0.f) || pv == INFINITY;             // what torch.multinomial rejects: NaN, +-inf, negative ...
        nonzero |= pv != 0.f;                               // ... or a zero sum
        s_key[i] = sid_topk_key(__fdiv_rn(pv, q[i]));
      }
      bad = __any_sync(0xffffffffu, bad);
      nonzero = __any_sync(0xffffffffu, nonzero);
      if (reject && lane == 0 && (bad || !nonzero)) atomicAdd(&reject[bad ? 0 : 1], 1);
    }
    __syncwarp();
    sid_warp_top_n(s_key, K, nc, s_hist, s_sk, s_si, s_tok + beam * nc, lane);
    sid_beam_mask<FILTER>(trie, ex, b, generated + row * h, h, K, s_mask, lane);
    const float plp = log_probas ? log_probas[row] : 0.f;
    for (int r = lane; r < nc; r += 32) {
      const int64_t tok = s_tok[beam * nc + r];
      if (WARP) {                                           // the model's log-probability; key 0: a filler outside N+
        const bool drawn = s_key[tok] != 0u;
        const float lp = drawn ? __fsub_rn(p[tok], lse) : -INFINITY;
        if (samples) samples[row * nc + r] = tok;
        if (samp_log_p) samp_log_p[row * nc + r] = lp;
        s_score[beam * nc + r] = sid_extension_score(drawn && sid_mask_has(s_mask, (int)tok), __fadd_rn(lp, plp));
      } else {
        const float lp = logf(p[tok]);
        if (samples) samples[row * nc + r] = tok;
        if (samp_log_p) samp_log_p[row * nc + r] = lp;
        s_score[beam * nc + r] = sid_extension_score(sid_mask_has(s_mask, (int)tok), lp + plp);
      }
      s_taken[beam * nc + r] = 0;
    }
  }
  __syncthreads();
  if constexpr (CAP) {
    // group of each beam (the lowest beam with the same len-prefix), then each candidate's rank in its group's order (score
    // descending, lowest flat index first): past m it drops to -inf.  s_taken marks the dropped ones until every rank is taken.
    int* s_grp = reinterpret_cast<int*>(s_taken + ((E + 3) & ~3));                                       // [kp]
    const int nt = blockDim.x;
    for (int t = threadIdx.x; t < kp; t += nt) {
      const int64_t* ids = generated + ((int64_t)b * kp + t) * h;
      int g = t;
      for (int j = 0; j < t && g == t; ++j) {
        const int64_t* jd = generated + ((int64_t)b * kp + j) * h;
        bool eq = true;
        for (int l = 0; l < cap.len; ++l) eq &= jd[l] == ids[l];
        if (eq) g = j;
      }
      s_grp[t] = g;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < E; e += nt) {
      const int g = s_grp[e / nc];
      const float sc = s_score[e];
      int above = 0;
      for (int j = g; j < kp && above < cap.m; ++j) {
        if (s_grp[j] != g) continue;
#pragma unroll 1
        for (int r = 0; r < nc; ++r) {
          const int f = j * nc + r;
          const float o = s_score[f];
          above += o > sc || (o == sc && f < e);
        }
      }
      s_taken[e] = above >= cap.m;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < E; e += nt) {
      if (s_taken[e]) {
        s_score[e] = -INFINITY;
        s_taken[e] = 0;
      }
    }
    __syncthreads();
  }
  if (w == 0)
    sid_keep_best(s_score, s_taken, s_tok, E, nc, b, kp, h, k, generated, out_generated, out_log_probas, out_parent, lane);
}

// The filter arguments of the *_excluding / *_including entry points: the arrays of rqb200_sid_exclusion_build /
// rqb200_sid_inclusion_build (count null: none).
static int sid_excl_of(const int* pos, const int64_t* keys, const int* count, int M, int H, int levels, const char* what,
                       SidExcl& ex, bool include = false) {
  ex = SidExcl{pos, reinterpret_cast<const long long*>(keys), count, M, H, include};
  if (!count) return RQB_OK;
  RQB_CHECK_ARG(pos && keys && M > 0 && M <= SID_EXCL_MAX_M && H >= levels && H <= RQB_MAX_LEVELS,
                "%s: bad %s (M = %d, H = %d, need M <= %d and H >= %d)", what, include ? "inclusion" : "exclusion", M, H,
                SID_EXCL_MAX_M, levels);
  return RQB_OK;
}

// The sampling temperature and nucleus mass of a warped draw: finite T > 0, 0 < top_p <= 1
static int sid_check_warp(float temp, float top_p, const char* what) {
  RQB_CHECK_ARG(temp > 0.f && temp < INFINITY && top_p > 0.f && top_p <= 1.f,
                "%s: need a finite temperature > 0 and 0 < top_p <= 1 (temperature = %g, top_p = %g)", what, (double)temp,
                (double)top_p);
  return RQB_OK;
}

// The per-prefix cap of a level h: 1 <= len <= h and m >= 1 (RQB_ERR_INVALID otherwise)
static int sid_check_cap(const SidCap& cap, int h, const char* what) {
  RQB_CHECK_ARG(cap.len >= 1 && cap.len <= h && cap.m >= 1,
                "%s: need 1 <= prefix_len <= h and max_per_prefix >= 1 (prefix_len = %d, h = %d, max_per_prefix = %d)", what,
                cap.len, h, cap.m);
  return RQB_OK;
}

// The filter of a *_capped entry point: mode (SidFilterMode), then the arrays of rqb200_sid_exclusion_build /
// rqb200_sid_inclusion_build (null / 0 without a filter)
static int sid_filter_of(int mode, const int* pos, const int64_t* keys, const int* count, int M, int H, int levels,
                         const char* what, SidExcl& f) {
  f = SidExcl{};
  RQB_CHECK_ARG(mode == SID_FILTER_NONE || mode == SID_FILTER_EXCLUDE || mode == SID_FILTER_INCLUDE, "%s: bad filter mode %d",
                what, mode);
  if (mode == SID_FILTER_NONE) return RQB_OK;
  RQB_CHECK_ARG(count, "%s: filter mode %d needs the filter's arrays", what, mode);
  return sid_excl_of(pos, keys, count, M, H, levels, what, f, mode == SID_FILTER_INCLUDE);
}

template <bool WARP>
static int sid_sample_select(const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride,
                             const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K,
                             const void* prefix_workspace, int64_t* out_generated, float* out_log_probas, int64_t* out_parent,
                             int64_t* samples, float* samp_log_p, int* reject, const SidExcl& ex, float temp, float top_p,
                             void* stream, const SidCap* cap = nullptr) {
  RQB_CHECK_ARG(B >= 0 && kp > 0 && nc > 0 && h >= 0 && h < C && C <= 8 && k > 0 && K > 0 && probas_stride >= K &&
                    noise_stride >= K, "sid_trie_sample_select: bad argument (B=%d kp=%d nc=%d h=%d k=%d C=%d K=%d)", B, kp, nc, h,
                k, C, K);
  if (WARP && sid_check_warp(temp, top_p, "sid_trie_sample_select_warped") != RQB_OK) return RQB_ERR_INVALID;
  if (cap && sid_check_cap(*cap, h, WARP ? "sid_trie_sample_select_warped_capped" : "sid_trie_sample_select_capped") != RQB_OK)
    return RQB_ERR_INVALID;
  if (nc > K || K > SID_SAMPLE_MAX_K || kp * nc > SID_BEAM_MAX_E || k > 32) {
    rqb_set_error("sid_trie_sample_select: need nc <= K <= %d, kp * nc <= %d, k <= 32 (nc = %d, K = %d, kp * nc = %d, k = %d)",
                  SID_SAMPLE_MAX_K, SID_BEAM_MAX_E, nc, K, kp * nc, k);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(probas && noise && prefix_workspace && out_generated && out_log_probas && out_parent && (h == 0 || generated) &&
                    (h == 0 || log_probas), "sid_trie_sample_select: null pointer");
  const int W = kp < SID_SAMPLE_MAX_WARPS ? kp : SID_SAMPLE_MAX_WARPS;
  const bool capped = cap && cap->m < k;                    // a cap of k or more cannot bind: the uncapped kernel
  size_t smem = sid_sample_smem<WARP>(kp, nc, K);
  if (capped) smem = (smem + 3) / 4 * 4 + (size_t)kp * sizeof(int);   // the beams' groups after s_taken
  const int mode = sid_filter_mode(ex);
  auto kernel = capped ? (mode == SID_FILTER_INCLUDE ? sid_sample_select_kernel<SID_FILTER_INCLUDE, WARP, true>
                          : mode == SID_FILTER_EXCLUDE ? sid_sample_select_kernel<SID_FILTER_EXCLUDE, WARP, true>
                                                       : sid_sample_select_kernel<SID_FILTER_NONE, WARP, true>)
                : mode == SID_FILTER_INCLUDE ? sid_sample_select_kernel<SID_FILTER_INCLUDE, WARP>
                : mode == SID_FILTER_EXCLUDE ? sid_sample_select_kernel<SID_FILTER_EXCLUDE, WARP>
                                             : sid_sample_select_kernel<SID_FILTER_NONE, WARP>;
  RQB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<B, W * 32, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      probas, probas_stride, noise, noise_stride, generated, log_probas, kp, nc, h, k, K,
      SidTrie{reinterpret_cast<const unsigned char*>(prefix_workspace), h + 1}, out_generated, out_log_probas, out_parent, samples,
      samp_log_p, reject, ex, temp, top_p, capped ? *cap : SidCap{0, 0});
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_sid_trie_sample_select(const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride,
                                             const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k,
                                             int C, int K, const void* prefix_workspace, int64_t* out_generated,
                                             float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p,
                                             int* reject, void* stream) {
  return sid_sample_select<false>(probas, probas_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                  prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, reject, SidExcl{},
                                  1.f, 1.f, stream);
}

extern "C" int rqb200_sid_trie_sample_select_excluding(
    const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* reject, const int* ex_pos,
    const int64_t* ex_blocked, const int* ex_count, int ex_M, int ex_H, void* stream) {
  SidExcl ex;
  const int rc = sid_excl_of(ex_pos, ex_blocked, ex_count, ex_M, ex_H, h + 1, "sid_trie_sample_select_excluding", ex);
  if (rc != RQB_OK) return rc;
  return sid_sample_select<false>(probas, probas_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                  prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, reject, ex, 1.f,
                                  1.f, stream);
}

extern "C" int rqb200_sid_trie_sample_select_including(
    const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* reject, const int* in_pos,
    const int64_t* in_keys, const int* in_count, int in_M, int in_H, void* stream) {
  SidExcl in;
  const int rc = sid_excl_of(in_pos, in_keys, in_count, in_M, in_H, h + 1, "sid_trie_sample_select_including", in, true);
  if (rc != RQB_OK) return rc;
  return sid_sample_select<false>(probas, probas_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                  prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, reject, in, 1.f,
                                  1.f, stream);
}

extern "C" int rqb200_sid_trie_sample_select_warped(const float* logits, int64_t logits_stride, const float* noise,
                                                    int64_t noise_stride, const int64_t* generated, const float* log_probas, int B,
                                                    int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace,
                                                    int64_t* out_generated, float* out_log_probas, int64_t* out_parent,
                                                    int64_t* samples, float* samp_log_p, int* bad, float temperature, float top_p,
                                                    void* stream) {
  return sid_sample_select<true>(logits, logits_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                 prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, bad, SidExcl{},
                                 temperature, top_p, stream);
}

extern "C" int rqb200_sid_trie_sample_select_warped_excluding(
    const float* logits, int64_t logits_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* bad, float temperature, float top_p,
    const int* ex_pos, const int64_t* ex_blocked, const int* ex_count, int ex_M, int ex_H, void* stream) {
  SidExcl ex;
  const int rc = sid_excl_of(ex_pos, ex_blocked, ex_count, ex_M, ex_H, h + 1, "sid_trie_sample_select_warped_excluding", ex);
  if (rc != RQB_OK) return rc;
  return sid_sample_select<true>(logits, logits_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                 prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, bad, ex,
                                 temperature, top_p, stream);
}

extern "C" int rqb200_sid_trie_sample_select_warped_including(
    const float* logits, int64_t logits_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* bad, float temperature, float top_p,
    const int* in_pos, const int64_t* in_keys, const int* in_count, int in_M, int in_H, void* stream) {
  SidExcl in;
  const int rc = sid_excl_of(in_pos, in_keys, in_count, in_M, in_H, h + 1, "sid_trie_sample_select_warped_including", in, true);
  if (rc != RQB_OK) return rc;
  return sid_sample_select<true>(logits, logits_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                 prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, bad, in,
                                 temperature, top_p, stream);
}

extern "C" int rqb200_sid_trie_sample_select_capped(
    const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* reject, int prefix_len, int max_per_prefix,
    int filter_mode, const int* f_pos, const int64_t* f_keys, const int* f_count, int f_M, int f_H, void* stream) {
  SidExcl f;
  const int rc = sid_filter_of(filter_mode, f_pos, f_keys, f_count, f_M, f_H, h + 1, "sid_trie_sample_select_capped", f);
  if (rc != RQB_OK) return rc;
  const SidCap cap{prefix_len, max_per_prefix};
  return sid_sample_select<false>(probas, probas_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                  prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, reject, f, 1.f,
                                  1.f, stream, &cap);
}

extern "C" int rqb200_sid_trie_sample_select_warped_capped(
    const float* logits, int64_t logits_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* bad, float temperature, float top_p,
    int prefix_len, int max_per_prefix, int filter_mode, const int* f_pos, const int64_t* f_keys, const int* f_count, int f_M,
    int f_H, void* stream) {
  SidExcl f;
  const int rc = sid_filter_of(filter_mode, f_pos, f_keys, f_count, f_M, f_H, h + 1, "sid_trie_sample_select_warped_capped", f);
  if (rc != RQB_OK) return rc;
  const SidCap cap{prefix_len, max_per_prefix};
  return sid_sample_select<true>(logits, logits_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                 prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, bad, f,
                                 temperature, top_p, stream, &cap);
}

// ---------------------------------------------------------------------------------------------------------------------
// One level of the exhaustive constrained beam search, from the head's logits, in one launch: every code of every beam is a
// candidate.  Per beam row lse = m + logf(sum expf(x - m)) in a fixed reduction order; candidate e = beam * K + c scores
// (x[c] - lse) + log_probas[beam], -inf when the extended prefix is not in the corpus or the score is NaN
// (sid_extension_score); the k largest are kept in descending order, equal scores by ascending e (sid_keep_best's rule).
// One CTA per batch row.  A candidate's order key is the sid_topk_key image of its score (-0 folded into +0) above the 16 bits
// 0xffff - e, so the E = kp * K <= 65 536 keys of a row are distinct and "the k largest keys" is exactly that order.  A
// block-wide radix selection (8-bit digits; it stops once the bin of the chosen digit holds exactly the entries still wanted)
// finds the smallest kept key, the k keys at or above it are collected and each is ranked among them.  The histograms are
// integer counts and the ranks compare distinct keys: no result depends on the order of atomics.  The 32-bit score keys stay
// in shared memory when E <= SID_TOPK_SMEM_KEYS; above that every pass recomputes them from the logits.  The score is written
// with explicit roundings (no contraction), so a recomputed key has the same bits as the first.  Every beam's children are
// first expanded into a K-bit mask in shared memory (sid_child_mask, after the keys), and a candidate's test is one bit test.
#define SID_TOPK_MAX_K 2048
#define SID_TOPK_MAX_BEAMS 32
#define SID_TOPK_MAX_THREADS 512
#define SID_TOPK_SMEM_KEYS (48 * 1024)

struct SidTopkShared {
  int hist[256];
  int ctl[3];                                               // chosen digit, entries above its bin, entries in its bin
  int nsel;
  float lse[SID_TOPK_MAX_BEAMS];
  float plp[SID_TOPK_MAX_BEAMS];
  int64_t gen[SID_TOPK_MAX_BEAMS * 7];                      // the beams' ids, [kp][h], h < C <= 8
  unsigned long long sel[32];
};

// candidate e's 32-bit score key; mask: the beams' child masks [kp][ceil(K / 32)]
__device__ __forceinline__ unsigned int sid_topk_candidate(const float* __restrict__ logits, int64_t ld, int64_t row0, int K, int e,
                                                           const SidTopkShared& s, const unsigned int* mask) {
  const int beam = e / K, c = e - beam * K;
  const float lp = __fadd_rn(__fsub_rn(logits[(row0 + beam) * ld + c], s.lse[beam]), s.plp[beam]);
  const float sc = sid_extension_score(sid_mask_has(mask + beam * ((K + 31) >> 5), c), lp);
  return sid_topk_key(sc == 0.f ? 0.f : sc);
}

#define SID_FILLER_KEY 0x007fffffu                          // sid_topk_key(-inf): below every other candidate's key

// byte offset of the CAP mode's per-beam arrays in sid_beam_topk_kernel's dynamic shared memory (after keys and masks), and
// their size: 2 x 64-bit cut + 4 ints per beam
__host__ __device__ __forceinline__ size_t sid_topk_cap_offset(int E, int kp, int K, bool keys_in_smem) {
  return ((size_t)((keys_in_smem ? E : 0) + kp * ((K + 31) / 32)) * sizeof(unsigned int) + 7) / 8 * 8;
}
#define SID_TOPK_CAP_BYTES_PER_BEAM (2 * sizeof(unsigned long long) + 4 * sizeof(int))

// Threads 0 .. kp - 1: grp[beam] = the lowest beam of the row whose first len ids equal beam's (ids [kp][h] in shared memory).
// Then beams 0 .. kp - 1 again: order[pos] = the beams by (group, beam), start[g] / count[g] = a leader g's run in `order`.
// Two __syncthreads; every thread must call.
__device__ __forceinline__ void sid_cap_groups(const int64_t* ids, int h, int kp, int len, int* grp, int* order, int* start,
                                               int* count) {
  const int t = threadIdx.x;
  if (t < kp) {
    int g = t;
    for (int j = 0; j < t && g == t; ++j) {
      bool eq = true;
      for (int l = 0; l < len; ++l) eq &= ids[j * h + l] == ids[t * h + l];
      if (eq) g = j;
    }
    grp[t] = g;
  }
  __syncthreads();
  if (t < kp) {
    const int g = grp[t];
    int pos = 0, n = 0, lead = 0;
    for (int j = 0; j < kp; ++j) {
      const int gj = grp[j];
      pos += gj < g || (gj == g && j < t);
      n += gj == g;
      lead += gj < g;
    }
    order[pos] = t;
    if (g == t) {
      start[t] = lead;
      count[t] = n;
    }
  }
  __syncthreads();
}

// The whole block: the cut (prefix, digit mask) of the `want` largest of the n distinct 48-bit keys key_at(i), i < n -- a key
// is among them iff (v & pmask) >= prefix -- by sid_beam_topk_kernel's radix selection.  s.hist is zero on entry and on return.
template <typename KeyAt>
__device__ __forceinline__ void sid_block_cut(const KeyAt& key_at, int n, int want, SidTopkShared& s, unsigned long long& prefix,
                                              unsigned long long& pmask) {
  const int nt = blockDim.x, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned int lt = (1u << lane) - 1u;
  prefix = 0;
  pmask = 0;
  for (int shift = 40; shift >= 0; shift -= 8) {
    for (int base = 0; base < n; base += nt) {
      const int i = base + threadIdx.x;
      int d = 256;
      if (i < n) {
        const unsigned long long v = key_at(i);
        if ((v & pmask) == prefix) d = (int)((v >> shift) & 255u);
      }
      const unsigned int same = __match_any_sync(0xffffffffu, d);
      if (d < 256 && (same & lt) == 0) atomicAdd(&s.hist[d], __popc(same));
    }
    __syncthreads();
    if (w == 0) {
      int c[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = s.hist[lane * 8 + j];
        s.hist[lane * 8 + j] = 0;
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
            s.ctl[0] = lane * 8 + j;
            s.ctl[1] = acc;
            s.ctl[2] = c[j];
            break;
          }
          acc += c[j];
        }
      }
    }
    __syncthreads();
    want -= s.ctl[1];
    prefix |= (unsigned long long)s.ctl[0] << shift;
    pmask |= 255ull << shift;
    if (s.ctl[2] == want) break;
  }
}

template <bool KEYS_IN_SMEM, int FILTER, bool CAP = false>  // FILTER: SidFilterMode; CAP: the per-prefix cap (SidCap)
__global__ void __launch_bounds__(SID_TOPK_MAX_THREADS) sid_beam_topk_kernel(
    const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ generated, const float* __restrict__ log_probas,
    int kp, int h, int k, int K, SidTrie trie, int64_t* __restrict__ out_generated, float* __restrict__ out_log_probas,
    int64_t* __restrict__ out_parent, int* __restrict__ bad, SidExcl ex, SidCap cap) {
  extern __shared__ __align__(16) unsigned char sid_smem[];
  __shared__ SidTopkShared s;
  unsigned int* s_key = reinterpret_cast<unsigned int*>(sid_smem);                // [E] when KEYS_IN_SMEM
  const int nt = blockDim.x, W = nt >> 5, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned int lt = (1u << lane) - 1u;
  const int b = blockIdx.x, E = kp * K;
  const int64_t row0 = (int64_t)b * kp;
  unsigned int* s_mask = s_key + (KEYS_IN_SMEM ? E : 0);   // [kp][ceil(K / 32)]
  // CAP: after the masks, per beam: the group's kept-key test (prefix, digit mask) at its leader, group, order, run start/count
  unsigned long long* s_cut = reinterpret_cast<unsigned long long*>(sid_smem + sid_topk_cap_offset(E, kp, K, KEYS_IN_SMEM));
  int* s_grp = reinterpret_cast<int*>(s_cut + 2 * kp);
  int* s_order = s_grp + kp;
  int* s_start = s_order + kp;
  int* s_count = s_start + kp;
  for (int i = threadIdx.x; i < 256; i += nt) s.hist[i] = 0;
  for (int i = threadIdx.x; i < kp * h; i += nt) s.gen[i] = generated[row0 * h + i];
  if (threadIdx.x == 0) s.nsel = 0;
  for (int beam = w; beam < kp; beam += W) {                // warp per beam: row maximum, then log-sum-exp
    const float* x = logits + (row0 + beam) * ld;
    float m = -INFINITY;
    bool odd = false;
    for (int c = lane; c < K; c += 32) {
      const float v = x[c];
      m = fmaxf(m, v);
      odd |= v != v || v == INFINITY;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    odd = __any_sync(0xffffffffu, odd);
    float sum = 0.f;
    for (int c = lane; c < K; c += 32) sum += expf(x[c] - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);   // every lane ends with the same bits
    if (lane == 0) {
      s.lse[beam] = m + logf(sum);                          // NaN for a row with NaN or +inf, or all -inf: its scores are -inf
      s.plp[beam] = log_probas ? log_probas[row0 + beam] : 0.f;
      if (bad && (odd || m == -INFINITY)) atomicAdd(bad, 1);
    }
  }
  __syncthreads();
  for (int beam = w; beam < kp; beam += W)
    sid_beam_mask<FILTER>(trie, ex, b, s.gen + beam * h, h, K, s_mask + beam * ((K + 31) >> 5), lane);
  __syncthreads();
  // CAP: candidate e's key, or the filler's when its group's cut leaves it out
  auto capped = [&](int e, unsigned int key) -> unsigned int {
    const int g = s_grp[e / K];
    const unsigned long long v = ((unsigned long long)key << 16) | (unsigned int)(0xffff - e);
    return (v & s_cut[2 * g + 1]) >= s_cut[2 * g] ? key : SID_FILLER_KEY;
  };
  if constexpr (CAP) {                                      // each group's cut: the radix selection over its beams' candidates
    sid_cap_groups(s.gen, h, kp, cap.len, s_grp, s_order, s_start, s_count);
    if (KEYS_IN_SMEM) {
      for (int e = threadIdx.x; e < E; e += nt) s_key[e] = sid_topk_candidate(logits, ld, row0, K, e, s, s_mask);
      __syncthreads();
    }
    for (int g = 0; g < kp; ++g) {
      if (s_grp[g] != g) continue;                          // uniform: every thread reads the same group table
      const int* members = s_order + s_start[g];
      auto key_at = [&](int i) -> unsigned long long {
        const int j = i / K;
        const int e = members[j] * K + (i - j * K);
        const unsigned int key = KEYS_IN_SMEM ? s_key[e] : sid_topk_candidate(logits, ld, row0, K, e, s, s_mask);
        return ((unsigned long long)key << 16) | (unsigned int)(0xffff - e);
      };
      unsigned long long cut, cut_mask;
      sid_block_cut(key_at, s_count[g] * K, cap.m, s, cut, cut_mask);
      if (threadIdx.x == 0) {
        s_cut[2 * g] = cut;
        s_cut[2 * g + 1] = cut_mask;
      }
    }
    __syncthreads();
    if (KEYS_IN_SMEM) {
      for (int e = threadIdx.x; e < E; e += nt) s_key[e] = capped(e, s_key[e]);
      __syncthreads();
    }
  }
  unsigned long long prefix = 0, pmask = 0;
  int want = k;                                             // entries still needed among those matching the decided digits
  for (int shift = 40; shift >= 0; shift -= 8) {
    for (int base = 0; base < E; base += nt) {
      const int e = base + threadIdx.x;
      int d = 256;
      if (e < E) {
        unsigned int key;
        if (KEYS_IN_SMEM) {
          if (shift == 40 && !CAP) s_key[e] = key = sid_topk_candidate(logits, ld, row0, K, e, s, s_mask);
          else key = s_key[e];
        } else {
          key = sid_topk_candidate(logits, ld, row0, K, e, s, s_mask);
          if (CAP) key = capped(e, key);
        }
        const unsigned long long v = ((unsigned long long)key << 16) | (unsigned int)(0xffff - e);
        if ((v & pmask) == prefix) d = (int)((v >> shift) & 255u);
      }
      const unsigned int same = __match_any_sync(0xffffffffu, d);
      if (d < 256 && (same & lt) == 0) atomicAdd(&s.hist[d], __popc(same));   // one add per distinct digit of the warp
    }
    __syncthreads();
    if (w == 0) {
      int c[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = s.hist[lane * 8 + j];
        s.hist[lane * 8 + j] = 0;                           // cleared for the next pass
        sum += c[j];
      }
      int suf = sum;                                        // entries in bins >= lane * 8
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
            s.ctl[0] = lane * 8 + j;
            s.ctl[1] = acc;
            s.ctl[2] = c[j];
            break;
          }
          acc += c[j];
        }
      }
    }
    __syncthreads();
    want -= s.ctl[1];
    prefix |= (unsigned long long)s.ctl[0] << shift;
    pmask |= 255ull << shift;
    if (s.ctl[2] == want) break;                            // the whole bin is kept: the threshold is decided
  }
  // the kept set: keys whose decided digits are above the prefix (k - want of them) or equal to it (want of them)
  for (int e = threadIdx.x; e < E; e += nt) {
    unsigned int key = KEYS_IN_SMEM ? s_key[e] : sid_topk_candidate(logits, ld, row0, K, e, s, s_mask);
    if (CAP && !KEYS_IN_SMEM) key = capped(e, key);
    const unsigned long long v = ((unsigned long long)key << 16) | (unsigned int)(0xffff - e);
    if ((v & pmask) >= prefix) s.sel[atomicAdd(&s.nsel, 1)] = v;
  }
  __syncthreads();
  if (threadIdx.x < k) {
    const unsigned long long v = s.sel[threadIdx.x];
    int r = 0;
    for (int q = 0; q < k; ++q) r += s.sel[q] > v;
    const unsigned int key = (unsigned int)(v >> 16);
    const int e = 0xffff - (int)(v & 0xffffu);
    const int beam = e / K;
    const int64_t o = (int64_t)b * k + r;
    out_log_probas[o] = __uint_as_float((key & 0x80000000u) ? key ^ 0x80000000u : ~key);   // sid_topk_key inverted
    out_parent[o] = row0 + beam;
    int64_t* g = out_generated + o * (h + 1);
    for (int j = 0; j < h; ++j) g[j] = s.gen[beam * h + j];
    g[h] = e - beam * K;
  }
}

template <int FILTER, bool CAP>
static int sid_beam_topk_launch(const float* logits, int64_t logits_stride, const int64_t* generated, const float* log_probas,
                                int B, int kp, int h, int k, int K, const SidTrie& trie, int64_t* out_generated,
                                float* out_log_probas, int64_t* out_parent, int* bad, const SidExcl& ex, const SidCap& cap,
                                cudaStream_t st) {
  const int E = kp * K;
  const int nt = E >= 4096 ? SID_TOPK_MAX_THREADS : E >= 1024 ? 256 : 128;
  const size_t mask = (size_t)kp * ((K + 31) / 32) * sizeof(unsigned int);
  if (E <= SID_TOPK_SMEM_KEYS) {
    const size_t smem = CAP ? sid_topk_cap_offset(E, kp, K, true) + kp * SID_TOPK_CAP_BYTES_PER_BEAM
                            : (size_t)E * sizeof(unsigned int) + mask;
    RQB_CUDA(cudaFuncSetAttribute(sid_beam_topk_kernel<true, FILTER, CAP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    sid_beam_topk_kernel<true, FILTER, CAP><<<B, nt, smem, st>>>(logits, logits_stride, generated, log_probas, kp, h, k, K, trie,
                                                                 out_generated, out_log_probas, out_parent, bad, ex, cap);
  } else {
    const size_t smem = CAP ? sid_topk_cap_offset(E, kp, K, false) + kp * SID_TOPK_CAP_BYTES_PER_BEAM : mask;
    sid_beam_topk_kernel<false, FILTER, CAP><<<B, nt, smem, st>>>(logits, logits_stride, generated, log_probas, kp, h, k, K, trie,
                                                                  out_generated, out_log_probas, out_parent, bad, ex, cap);
  }
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

static int sid_beam_topk(const float* logits, int64_t logits_stride, const int64_t* generated, const float* log_probas, int B, int kp,
                         int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                         int64_t* out_parent, int* bad, const SidExcl& ex, void* stream, const SidCap* cap = nullptr) {
  RQB_CHECK_ARG(B >= 0 && kp > 0 && h >= 0 && h < C && C <= 8 && k > 0 && K > 0 && logits_stride >= K,
                "sid_trie_beam_topk: bad argument (B=%d kp=%d h=%d k=%d C=%d K=%d)", B, kp, h, k, C, K);
  if (cap && sid_check_cap(*cap, h, "sid_trie_beam_topk_capped") != RQB_OK) return RQB_ERR_INVALID;
  if (K > SID_TOPK_MAX_K || k > 32 || k > K || kp > SID_TOPK_MAX_BEAMS) {
    rqb_set_error("sid_trie_beam_topk: need K <= %d, k <= 32, k <= K, kp <= %d (K = %d, k = %d, kp = %d)", SID_TOPK_MAX_K,
                  SID_TOPK_MAX_BEAMS, K, k, kp);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(logits && prefix_workspace && out_generated && out_log_probas && out_parent && (h == 0 || generated) &&
                    (h == 0 || log_probas), "sid_trie_beam_topk: null pointer");
  const SidTrie trie{reinterpret_cast<const unsigned char*>(prefix_workspace), h + 1};
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const SidCap c = cap ? *cap : SidCap{0, 0};
  if (cap && cap->m < k) {                                  // a cap of k or more cannot bind: the uncapped kernel
    switch (sid_filter_mode(ex)) {
      case SID_FILTER_INCLUDE:
        return sid_beam_topk_launch<SID_FILTER_INCLUDE, true>(logits, logits_stride, generated, log_probas, B, kp, h, k, K, trie,
                                                              out_generated, out_log_probas, out_parent, bad, ex, c, st);
      case SID_FILTER_EXCLUDE:
        return sid_beam_topk_launch<SID_FILTER_EXCLUDE, true>(logits, logits_stride, generated, log_probas, B, kp, h, k, K, trie,
                                                              out_generated, out_log_probas, out_parent, bad, ex, c, st);
      default:
        return sid_beam_topk_launch<SID_FILTER_NONE, true>(logits, logits_stride, generated, log_probas, B, kp, h, k, K, trie,
                                                           out_generated, out_log_probas, out_parent, bad, ex, c, st);
    }
  }
  switch (sid_filter_mode(ex)) {
    case SID_FILTER_INCLUDE:
      return sid_beam_topk_launch<SID_FILTER_INCLUDE, false>(logits, logits_stride, generated, log_probas, B, kp, h, k, K, trie,
                                                             out_generated, out_log_probas, out_parent, bad, ex, c, st);
    case SID_FILTER_EXCLUDE:
      return sid_beam_topk_launch<SID_FILTER_EXCLUDE, false>(logits, logits_stride, generated, log_probas, B, kp, h, k, K, trie,
                                                             out_generated, out_log_probas, out_parent, bad, ex, c, st);
    default:
      return sid_beam_topk_launch<SID_FILTER_NONE, false>(logits, logits_stride, generated, log_probas, B, kp, h, k, K, trie,
                                                          out_generated, out_log_probas, out_parent, bad, ex, c, st);
  }
}

extern "C" int rqb200_sid_trie_beam_topk(const float* logits, int64_t logits_stride, const int64_t* generated, const float* log_probas,
                                         int B, int kp, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
                                         float* out_log_probas, int64_t* out_parent, int* bad, void* stream) {
  return sid_beam_topk(logits, logits_stride, generated, log_probas, B, kp, h, k, C, K, prefix_workspace, out_generated,
                       out_log_probas, out_parent, bad, SidExcl{}, stream);
}

extern "C" int rqb200_sid_trie_beam_topk_excluding(const float* logits, int64_t logits_stride, const int64_t* generated,
                                                   const float* log_probas, int B, int kp, int h, int k, int C, int K,
                                                   const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                                   int64_t* out_parent, int* bad, const int* ex_pos, const int64_t* ex_blocked,
                                                   const int* ex_count, int ex_M, int ex_H, void* stream) {
  SidExcl ex;
  const int rc = sid_excl_of(ex_pos, ex_blocked, ex_count, ex_M, ex_H, h + 1, "sid_trie_beam_topk_excluding", ex);
  if (rc != RQB_OK) return rc;
  return sid_beam_topk(logits, logits_stride, generated, log_probas, B, kp, h, k, C, K, prefix_workspace, out_generated,
                       out_log_probas, out_parent, bad, ex, stream);
}

extern "C" int rqb200_sid_trie_beam_topk_including(const float* logits, int64_t logits_stride, const int64_t* generated,
                                                   const float* log_probas, int B, int kp, int h, int k, int C, int K,
                                                   const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                                   int64_t* out_parent, int* bad, const int* in_pos, const int64_t* in_keys,
                                                   const int* in_count, int in_M, int in_H, void* stream) {
  SidExcl in;
  const int rc = sid_excl_of(in_pos, in_keys, in_count, in_M, in_H, h + 1, "sid_trie_beam_topk_including", in, true);
  if (rc != RQB_OK) return rc;
  return sid_beam_topk(logits, logits_stride, generated, log_probas, B, kp, h, k, C, K, prefix_workspace, out_generated,
                       out_log_probas, out_parent, bad, in, stream);
}

extern "C" int rqb200_sid_trie_beam_topk_capped(const float* logits, int64_t logits_stride, const int64_t* generated,
                                                const float* log_probas, int B, int kp, int h, int k, int C, int K,
                                                const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                                int64_t* out_parent, int* bad, int prefix_len, int max_per_prefix, int filter_mode,
                                                const int* f_pos, const int64_t* f_keys, const int* f_count, int f_M, int f_H,
                                                void* stream) {
  SidExcl f;
  const int rc = sid_filter_of(filter_mode, f_pos, f_keys, f_count, f_M, f_H, h + 1, "sid_trie_beam_topk_capped", f);
  if (rc != RQB_OK) return rc;
  const SidCap cap{prefix_len, max_per_prefix};
  return sid_beam_topk(logits, logits_stride, generated, log_probas, B, kp, h, k, C, K, prefix_workspace, out_generated,
                       out_log_probas, out_parent, bad, f, stream, &cap);
}

// ---------------------------------------------------------------------------------------------------------------------
// Corpus item table: from a generated id tuple back to the corpus items (rows) that carry it.  Row n of the corpus table
// [N, C] is item n; rows with equal tuples are told apart by their dedup rank (the tokeniser's last column: the number of
// earlier rows with the same tuple).  The build sorts the rows on their packed tuple with the trie's stable LSD radix sort
// (sid_sort_rows; a row holding an id outside [0, K) sorts last and is never retrievable), flags the first row of each distinct
// tuple, numbers the tuples with one scan and keeps
//   row[N]        the row ids in sorted order: equal tuples in ascending row order, i.e. dedup rank 0, 1, 2, ...;
//   key[U][G]     the U distinct retrievable tuples, packed as the sort packs them (G 64-bit words of `cols` ids each), ascending;
//   start[U + 1]  tuple u's rows are row[start[u] .. start[u + 1]).
// A lookup packs its tuple and binary-searches the keys.  A header at the start of the workspace locates the arrays.
//   workspace layout: header | row (int [N]) | key (u64 [N * G]) | start (int [N + 1]) | the sort's scratch (SidSortScratch),
//   256-byte aligned regions.
struct SidItemsHeader {
  int C, K;
  long long N;
  int U;                                                    // distinct retrievable tuples (written by the build)
  int G, width, cols;                                       // words per packed tuple, bits per id, ids per word
  unsigned long long row, key, start;                       // byte offsets
};

struct SidItemsLayout {
  SidItemsHeader h;
  SidSortScratch sort;                                      // sort.end: the workspace bytes
};

#define SID_ITEMS_MAX_G 3                                   // C <= 8 ids of at most 17 bits: 3 ids per word
#define SID_ITEMS_MAX_K 1024
#define SID_ITEMS_MAX_N 4096

static int sid_items_layout(int64_t N, int C, int K, SidItemsLayout& t) {
  if (N < 0 || N >= 0x7fffffffll || C <= 0 || C > 8 || K <= 0 || K > 65536) return 1;
  t = SidItemsLayout{};
  t.h.width = sid_id_bits(K);
  t.h.cols = 64 / t.h.width;
  t.h.C = C;
  t.h.K = K;
  t.h.N = N;
  t.h.G = (C + t.h.cols - 1) / t.h.cols;
  size_t at = sid_align256(sizeof(SidItemsHeader));
  t.h.row = at;
  at += sid_align256((size_t)N * sizeof(int));
  t.h.key = at;
  at += sid_align256((size_t)N * t.h.G * sizeof(unsigned long long));
  t.h.start = at;
  at += sid_align256(((size_t)N + 1) * sizeof(int));
  return sid_sort_scratch(N, 1, at, t.sort) ? 2 : 0;
}

extern "C" size_t rqb200_sid_items_workspace_bytes(int64_t N, int C, int K) {
  SidItemsLayout t;
  return sid_items_layout(N, C, K, t) ? 0 : t.sort.end;
}

// Byte offsets of the row[N] and start[N + 1] arrays in an item table's workspace (host arithmetic, no device): the exact
// ranking expands its chosen tuples to items through them.  Nonzero outside the table's limits.
extern "C" int rqb200_sid_items_offsets(int64_t N, int C, int K, size_t* row, size_t* start) {
  SidItemsLayout t;
  RQB_CHECK_ARG(row && start, "sid_items_offsets: null pointer");
  if (sid_items_layout(N, C, K, t) == 1) {                  // 2 (no device to size the sort's scratch) still lays out both
    rqb_set_error("sid_items_offsets: N = %lld, C = %d, K = %d is outside the item table's limits", (long long)N, C, K);
    return RQB_ERR_UNSUPPORTED;
  }
  *row = t.h.row;
  *start = t.h.start;
  return RQB_OK;
}

__global__ void sid_items_header_kernel(SidItemsHeader h, unsigned char* ws) {
  *reinterpret_cast<SidItemsHeader*>(ws) = h;               // U = 0 and start[0] = 0: the fill pass overwrites both when a row is valid
  reinterpret_cast<int*>(ws + h.start)[0] = 0;
}

// flag[r] = sorted row r is retrievable and its tuple differs from sorted row r - 1's (the unretrievable rows sort last)
__global__ void sid_items_flag_kernel(const int64_t* __restrict__ ids, int N, int C, int K, const int* __restrict__ perm,
                                      int* __restrict__ flag) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < N; r += gridDim.x * blockDim.x) {
    const int64_t* row = ids + (int64_t)perm[r] * C;
    bool f = sid_row_depth(row, C, K) == C;
    if (f && r > 0) {
      const int64_t* prev = ids + (int64_t)perm[r - 1] * C;
      bool same = true;
      for (int c = 0; c < C; ++c) same = same && prev[c] == row[c];
      f = !same;
    }
    flag[r] = f ? 1 : 0;
  }
}

// row[r] = perm[r]; the row starting tuple u = scan[r] - 1 writes key[u] and start[u]; the last retrievable row closes start[U]
// and stores U
__global__ void sid_items_fill_kernel(const int64_t* __restrict__ ids, int N, const int* __restrict__ perm, const int* __restrict__ flag,
                                      const int* __restrict__ scan, unsigned char* ws) {
  SidItemsHeader* hdr = reinterpret_cast<SidItemsHeader*>(ws);
  const int C = hdr->C, K = hdr->K, G = hdr->G, width = hdr->width, cols = hdr->cols;
  int* row_out = reinterpret_cast<int*>(ws + hdr->row);
  unsigned long long* key = reinterpret_cast<unsigned long long*>(ws + hdr->key);
  int* start = reinterpret_cast<int*>(ws + hdr->start);
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < N; r += gridDim.x * blockDim.x) {
    const int64_t* row = ids + (int64_t)perm[r] * C;
    row_out[r] = perm[r];
    if (sid_row_depth(row, C, K) < C) continue;
    const int s = scan[r];
    if (flag[r]) {
      for (int g = 0; g < G; ++g) key[(int64_t)(s - 1) * G + g] = sid_pack_cols(row, C, g * cols, min(C, (g + 1) * cols), width, K);
      start[s - 1] = r;
    }
    if (r == N - 1 || sid_row_depth(ids + (int64_t)perm[r + 1] * C, C, K) < C) {
      start[s] = r + 1;
      hdr->U = s;
    }
  }
}

extern "C" int rqb200_sid_items_build(const int64_t* cached_ids, int64_t N, int C, int K, void* workspace, size_t ws_bytes, void* stream) {
  RQB_CHECK_ARG(N >= 0 && C > 0 && K > 0 && workspace, "sid_items_build: bad argument");
  SidItemsLayout t;
  const int rc = sid_items_layout(N, C, K, t);
  if (rc == 1) {
    rqb_set_error("sid_items_build: need C <= 8, K <= 65536 and N < 2^31 - 1 (N = %lld, C = %d, K = %d)", (long long)N, C, K);
    return RQB_ERR_UNSUPPORTED;
  }
  if (rc == 2) {
    rqb_set_error("sid_items_build: the sort's workspace query failed (no CUDA device?)");
    return RQB_ERR_CUDA;
  }
  if (ws_bytes < t.sort.end) {
    rqb_set_error("sid_items_build: workspace too small");
    return RQB_ERR_WORKSPACE;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  sid_items_header_kernel<<<1, 1, 0, st>>>(t.h, ws);
  RQB_LAUNCH_CHECK();
  if (N == 0) return RQB_OK;
  RQB_CHECK_ARG(cached_ids, "sid_items_build: null pointer");
  const int n = (int)N;
  int grid = (n + 255) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  int* flag = reinterpret_cast<int*>(ws + t.sort.flag);
  int* scan = reinterpret_cast<int*>(ws + t.sort.scan);
  int* sorted = nullptr;
  const int sc = sid_sort_rows(cached_ids, n, C, K, true, ws, t.sort, grid, st, sorted);
  if (sc != RQB_OK) return sc;
  sid_items_flag_kernel<<<grid, 256, 0, st>>>(cached_ids, n, C, K, sorted, flag);
  RQB_LAUNCH_CHECK();
  size_t temp_bytes = t.sort.temp_bytes;
  RQB_CUDA(cub::DeviceScan::InclusiveSum(ws + t.sort.temp, temp_bytes, flag, scan, n, st));
  sid_items_fill_kernel<<<grid, 256, 0, st>>>(cached_ids, n, sorted, flag, scan, ws);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// lexicographic order of the G-word packed tuples m and q: -1, 0 or 1
__device__ __forceinline__ int sid_items_cmp(const unsigned long long* m, const unsigned long long (&q)[SID_ITEMS_MAX_G], int G) {
  int cmp = 0;
#pragma unroll
  for (int g = 0; g < SID_ITEMS_MAX_G; ++g) {
    if (cmp == 0 && g < G) {
      const unsigned long long v = __ldg(m + g);
      cmp = v < q[g] ? -1 : v > q[g] ? 1 : 0;
    }
  }
  return cmp;
}

// tuple u of the table whose C ids equal t[0, C) (C = the table's), or -1 (an id outside [0, K), or not in the corpus)
__device__ __forceinline__ int sid_items_find(const unsigned char* ws, const SidItemsHeader& h, const int64_t* t) {
  unsigned long long q[SID_ITEMS_MAX_G];
  for (int c = 0; c < h.C; ++c)
    if (t[c] < 0 || t[c] >= h.K) return -1;
#pragma unroll
  for (int g = 0; g < SID_ITEMS_MAX_G; ++g)
    q[g] = g < h.G ? sid_pack_cols(t, h.C, g * h.cols, min(h.C, (g + 1) * h.cols), h.width, h.K) : 0ull;
  const unsigned long long* key = reinterpret_cast<const unsigned long long*>(ws + h.key);
  int a = 0, b = h.U;                                       // first key >= q
  while (a < b) {
    const int mid = (a + b) >> 1;
    if (sid_items_cmp(key + (int64_t)mid * h.G, q, h.G) < 0) a = mid + 1;
    else b = mid;
  }
  return (a < h.U && sid_items_cmp(key + (int64_t)a * h.G, q, h.G) == 0) ? a : -1;
}

__global__ void sid_items_lookup_kernel(const unsigned char* __restrict__ ws, const int64_t* __restrict__ ids, int64_t stride, int64_t P,
                                        int with_dedup, int64_t* __restrict__ out) {
  const SidItemsHeader h = *reinterpret_cast<const SidItemsHeader*>(ws);
  const int* row = reinterpret_cast<const int*>(ws + h.row);
  const int* start = reinterpret_cast<const int*>(ws + h.start);
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t* t = ids + p * stride;
    const int u = sid_items_find(ws, h, t);
    int64_t item = -1;
    if (u >= 0) {
      const int64_t d = with_dedup ? t[h.C] : 0;
      const int s = __ldg(start + u), count = __ldg(start + u + 1) - s;
      if (d >= 0 && d < count) item = __ldg(row + s + d);
    }
    out[p] = item;
  }
}

extern "C" int rqb200_sid_items_lookup(const void* workspace, const int64_t* ids, int64_t ids_stride, int64_t P, int with_dedup,
                                       int64_t* out_item, void* stream) {
  RQB_CHECK_ARG(P >= 0 && ids_stride > 0, "sid_items_lookup: bad argument (P = %lld, stride = %lld)", (long long)P,
                (long long)ids_stride);
  if (P == 0) return RQB_OK;
  RQB_CHECK_ARG(workspace && ids && out_item, "sid_items_lookup: null pointer");
  int grid = (int)((P + 255) / 256);
  if (grid > 132 * 16) grid = 132 * 16;
  sid_items_lookup_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const unsigned char*>(workspace), ids, ids_stride, P, with_dedup, out_item);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// One CTA per history b: each beam that is finite (log_probas null, or above -inf) and whose tuple is in the corpus resolves to
// tuple u; a beam whose tuple an earlier beam carries counts 0 items, every other resolved beam its tuple's row count; an
// exclusive block scan of the k counts places each beam's rows, in beam order, and output slot o takes the row of the beam
// whose range holds it (a binary search in the scanned offsets).  No result depends on the order of atomics.  With an exclusion a
// beam skips its tuple's excluded rows; with an allow-list its tuple's rows are the eligible positions in [start[u], start[u + 1])
// (two binary searches), and its d-th item is the d-th of them.
#define SID_ITEMS_THREADS 256
#define SID_ITEMS_PER_THREAD (SID_ITEMS_MAX_K / SID_ITEMS_THREADS)

template <bool INCLUDE>                                     // with an allow-list (else no filter or an exclusion, as ex says)
__global__ void __launch_bounds__(SID_ITEMS_THREADS) sid_items_retrieve_kernel(
    const unsigned char* __restrict__ ws, const int64_t* __restrict__ generated, const float* __restrict__ log_probas, int k, int C,
    int n, int64_t* __restrict__ out_items, int* __restrict__ out_beam, int* __restrict__ out_count, SidExcl ex) {
  using Scan = cub::BlockScan<int, SID_ITEMS_THREADS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ int s_u[SID_ITEMS_MAX_K];
  __shared__ int s_off[SID_ITEMS_MAX_K + 1];
  __shared__ int s_first[INCLUDE ? SID_ITEMS_MAX_K : 1];   // INCLUDE: each beam's first eligible position's index in xp
  const SidItemsHeader h = *reinterpret_cast<const SidItemsHeader*>(ws);
  const int* row = reinterpret_cast<const int*>(ws + h.row);
  const int* start = reinterpret_cast<const int*>(ws + h.start);
  const int b = blockIdx.x;
  const int* xp = INCLUDE || ex.on() ? ex.pos_of(b) : nullptr;   // the history's excluded (INCLUDE: eligible) positions, ascending
  const int nx = INCLUDE || ex.on() ? ex.npos(b) : 0;
  for (int j = threadIdx.x; j < k; j += SID_ITEMS_THREADS) {
    const int64_t bj = (int64_t)b * k + j;
    const bool live = log_probas == nullptr || log_probas[bj] > -INFINITY;   // NaN is not above -inf either
    s_u[j] = (live && C == h.C) ? sid_items_find(ws, h, generated + bj * C) : -1;
  }
  __syncthreads();
  int cnt[SID_ITEMS_PER_THREAD];
#pragma unroll
  for (int i = 0; i < SID_ITEMS_PER_THREAD; ++i) {
    const int j = threadIdx.x * SID_ITEMS_PER_THREAD + i;
    cnt[i] = 0;
    if (j < k && s_u[j] >= 0) {
      const int u = s_u[j];
      bool seen = false;
      for (int q = 0; q < j && !seen; ++q) seen = s_u[q] == u;
      if (!seen) {
        const int s = __ldg(start + u), e = __ldg(start + u + 1);
        if (INCLUDE) {
          s_first[j] = sid_lower_bound(xp, nx, s);
          cnt[i] = sid_lower_bound(xp, nx, e) - s_first[j];
        } else {
          cnt[i] = e - s - (xp ? sid_excluded_in(xp, nx, s, e) : 0);
        }
      }
    }
  }
  int off[SID_ITEMS_PER_THREAD], total;
  Scan(scan_tmp).ExclusiveSum(cnt, off, total);
#pragma unroll
  for (int i = 0; i < SID_ITEMS_PER_THREAD; ++i) {
    const int j = threadIdx.x * SID_ITEMS_PER_THREAD + i;
    if (j < k) s_off[j] = off[i];
  }
  if (threadIdx.x == 0) s_off[k] = total;
  __syncthreads();
  const int m = min(total, n);
  for (int o = threadIdx.x; o < n; o += SID_ITEMS_THREADS) {
    int64_t item = -1;
    int beam = -1;
    if (o < m) {                                            // s_off[lo] <= o < s_off[hi]: beam lo holds slot o
      int lo = 0, hi = k;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_off[mid] <= o) lo = mid;
        else hi = mid;
      }
      beam = lo;
      const int d = o - s_off[lo];
      if (INCLUDE) {
        item = __ldg(row + xp[s_first[lo] + d]);
      } else {
        const int s = __ldg(start + s_u[lo]);
        item = __ldg(row + (xp ? sid_nth_kept(xp, nx, s, d) : s + d));
      }
    }
    out_items[(int64_t)b * n + o] = item;
    out_beam[(int64_t)b * n + o] = beam;
  }
  if (threadIdx.x == 0) out_count[b] = m;
}

static int sid_items_retrieve(const void* workspace, const int64_t* generated, const float* log_probas, int B, int k, int C, int n,
                              int64_t* out_items, int* out_beam, int* out_count, const SidExcl& ex, void* stream) {
  RQB_CHECK_ARG(B >= 0 && k > 0 && C > 0 && n > 0, "sid_items_retrieve: bad argument (B = %d, k = %d, C = %d, n = %d)", B, k, C, n);
  if (k > SID_ITEMS_MAX_K || n > SID_ITEMS_MAX_N) {
    rqb_set_error("sid_items_retrieve: need k <= %d and n <= %d (k = %d, n = %d)", SID_ITEMS_MAX_K, SID_ITEMS_MAX_N, k, n);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(workspace && generated && out_items && out_beam && out_count, "sid_items_retrieve: null pointer");
  auto kernel = sid_filter_mode(ex) == SID_FILTER_INCLUDE ? sid_items_retrieve_kernel<true> : sid_items_retrieve_kernel<false>;
  kernel<<<B, SID_ITEMS_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const unsigned char*>(workspace), generated, log_probas, k, C, n, out_items, out_beam, out_count, ex);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_sid_items_retrieve(const void* workspace, const int64_t* generated, const float* log_probas, int B, int k, int C,
                                         int n, int64_t* out_items, int* out_beam, int* out_count, void* stream) {
  return sid_items_retrieve(workspace, generated, log_probas, B, k, C, n, out_items, out_beam, out_count, SidExcl{}, stream);
}

extern "C" int rqb200_sid_items_retrieve_excluding(const void* workspace, const int64_t* generated, const float* log_probas, int B,
                                                   int k, int C, int n, int64_t* out_items, int* out_beam, int* out_count,
                                                   const int* ex_pos, const int64_t* ex_blocked, const int* ex_count, int ex_M,
                                                   int ex_H, void* stream) {
  SidExcl ex;
  const int rc = sid_excl_of(ex_pos, ex_blocked, ex_count, ex_M, ex_H, 0, "sid_items_retrieve_excluding", ex);
  if (rc != RQB_OK) return rc;
  return sid_items_retrieve(workspace, generated, log_probas, B, k, C, n, out_items, out_beam, out_count, ex, stream);
}

extern "C" int rqb200_sid_items_retrieve_including(const void* workspace, const int64_t* generated, const float* log_probas, int B,
                                                   int k, int C, int n, int64_t* out_items, int* out_beam, int* out_count,
                                                   const int* in_pos, const int64_t* in_keys, const int* in_count, int in_M,
                                                   int in_H, void* stream) {
  SidExcl in;
  const int rc = sid_excl_of(in_pos, in_keys, in_count, in_M, in_H, 0, "sid_items_retrieve_including", in, true);
  if (rc != RQB_OK) return rc;
  return sid_items_retrieve(workspace, generated, log_probas, B, k, C, n, out_items, out_beam, out_count, in, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// Per-history exclusion sets (csrc/sid_excl.cuh for the layout): "do not return these items" for the search kernels above, the
// item retrieval and the exact ranking's selection.  One CTA per history over its M entries (items, -1 pads): each item maps to
// its sorted position in the item table (inv, the inverse of the table's row array; positions from start[U] on are unretrievable
// rows and dropped), a block radix sort orders the positions and a block scan drops repeats.  The table's order is
// lexicographic, so the excluded items under an l-prefix p are one run of the sorted positions, and p's retrievable rows are
// start[lo] .. start[hi] with [lo, hi) the leaves whose keys (leaf_key, the packed tuples of the table's U leaves, ascending)
// begin with p: two binary searches.  The first position of each run flags p as blocked when the run covers all those rows;
// a block scan per level numbers the blocked prefixes.  Plain stores to distinct addresses; the cost depends on M and H only.
//
// Per-history allow-lists ("return only these items") come from the same body (INCLUDE): the positions are sorted and
// de-duplicated alike, those found in an exclusion's sorted positions (ex, one binary search each) are dropped as well, and the
// first position of each run flags its l-prefix as valid, so each level's keys are the distinct l-prefixes of the eligible
// positions, ascending because the positions are.
#define SID_EXCL_THREADS 512

template <int IPT, bool INCLUDE>
__global__ void __launch_bounds__(SID_EXCL_THREADS) sid_filter_kernel(
    const int64_t* __restrict__ items, int M, int64_t N, const int* __restrict__ inv, const int* __restrict__ start,
    const long long* __restrict__ leaf_key, int U, int H, int K, int* __restrict__ pos, long long* __restrict__ blocked,
    int* __restrict__ count, SidExcl ex) {
  using Sort = cub::BlockRadixSort<unsigned int, SID_EXCL_THREADS, IPT>;
  using Scan = cub::BlockScan<int, SID_EXCL_THREADS>;
  __shared__ union {
    typename Sort::TempStorage sort;
    typename Scan::TempStorage scan;
  } tmp;
  __shared__ int s_pos[SID_EXCL_THREADS * IPT];
  __shared__ unsigned int s_last[SID_EXCL_THREADS];
  __shared__ long long s_last_key[SID_EXCL_THREADS];
  __shared__ int s_bad;
  const unsigned int none = 0xffffffffu;
  const int64_t b = blockIdx.x;
  const int tid = threadIdx.x;
  const int n_items = U > 0 ? __ldg(start + U) : 0;
  if (tid == 0) s_bad = 0;
  unsigned int key[IPT];
  int bad = 0;
#pragma unroll
  for (int j = 0; j < IPT; ++j) {                           // blocked: thread t holds entries t IPT .. t IPT + IPT - 1
    const int c = tid * IPT + j;
    key[j] = none;
    if (c < M) {
      const int64_t v = items[b * M + c];
      if (v < -1 || v >= N) ++bad;
      else if (v >= 0) {
        const int r = __ldg(inv + v);
        if (r < n_items) key[j] = (unsigned int)r;
      }
    }
  }
  Sort(tmp.sort).Sort(key);
  __syncthreads();
  s_last[tid] = key[IPT - 1];
  if (bad) atomicAdd(&s_bad, bad);                          // an integer count: its value does not depend on the order
  __syncthreads();
  int flag[IPT], idx[IPT], total;
#pragma unroll
  for (int j = 0; j < IPT; ++j) {
    const unsigned int prev = j > 0 ? key[j - 1] : tid > 0 ? s_last[tid - 1] : none;
    flag[j] = key[j] != none && key[j] != prev ? 1 : 0;
    if (INCLUDE && flag[j] && ex.on()) {                    // an excluded position is not eligible
      const int* xp = ex.pos_of(b);
      const int nx = ex.npos(b), at = sid_lower_bound(xp, nx, (int)key[j]);
      if (at < nx && xp[at] == (int)key[j]) flag[j] = 0;
    }
  }
  Scan(tmp.scan).InclusiveSum(flag, idx, total);
  __syncthreads();
#pragma unroll
  for (int j = 0; j < IPT; ++j)
    if (flag[j]) s_pos[idx[j] - 1] = (int)key[j];
  __syncthreads();
  int* out_pos = pos + b * M;
  for (int i = tid; i < M; i += SID_EXCL_THREADS) out_pos[i] = i < total ? s_pos[i] : -1;
  long long lk[IPT];                                        // the leaf key of distinct position i = t IPT + j
#pragma unroll
  for (int j = 0; j < IPT; ++j) {
    const int i = tid * IPT + j;
    lk[j] = -1;
    if (i < total) {
      int lo = 0, hi = U;                                   // the leaf u with start[u] <= position < start[u + 1]
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(start + mid) <= s_pos[i]) lo = mid;
        else hi = mid;
      }
      lk[j] = __ldg(leaf_key + lo);
    }
  }
  s_last_key[tid] = lk[IPT - 1];
  __syncthreads();
  const long long prev_key = tid > 0 ? s_last_key[tid - 1] : -1;
  int* out_count = count + b * (H + 2);
  long long div = 1;                                        // K^(H - l): a leaf key over div is its l-prefix's key
  for (int l = 1; l < H; ++l) div *= K;
  for (int l = 1; l <= H; ++l) {
    long long p[IPT];
#pragma unroll
    for (int j = 0; j < IPT; ++j) {
      const int i = tid * IPT + j;
      p[j] = i < total ? lk[j] / div : -1;
      flag[j] = 0;
      const long long before = j > 0 ? lk[j - 1] : prev_key;
      if (i < total && (before < 0 || before / div != p[j])) {   // the first position under prefix p[j]
        if (INCLUDE) {
          flag[j] = 1;
        } else {
          const int lo = sid_lower_bound(leaf_key, U, p[j] * div), hi = sid_lower_bound(leaf_key, U, (p[j] + 1) * div);
          const int s = __ldg(start + lo), e = __ldg(start + hi);
          flag[j] = sid_lower_bound(s_pos, total, e) - i == e - s ? 1 : 0;
        }
      }
    }
    int nb;
    Scan(tmp.scan).InclusiveSum(flag, idx, nb);
    __syncthreads();                                        // scan storage is reused by the next level
    long long* out_blocked = blocked + (b * H + (l - 1)) * M;
#pragma unroll
    for (int j = 0; j < IPT; ++j)
      if (flag[j]) out_blocked[idx[j] - 1] = p[j];
    for (int i = nb + tid; i < M; i += SID_EXCL_THREADS) out_blocked[i] = -1;
    if (tid == 0) out_count[l] = nb;
    div /= K;
  }
  if (tid == 0) {
    out_count[0] = total;
    out_count[H + 1] = s_bad;
  }
}

static int sid_filter_build(const int64_t* items, int B, int M, int64_t N, const int* inv, const int* start, const int64_t* leaf_key,
                            int U, int H, int K, int* pos, int64_t* keys, int* count, const SidExcl& ex, bool include,
                            const char* what, void* stream) {
  RQB_CHECK_ARG(B >= 0 && M > 0 && N >= 0 && N < 0x7fffffffll && U >= 0 && U <= N && H > 0 && K > 0,
                "%s: bad argument (B = %d, M = %d, N = %lld, U = %d, H = %d, K = %d)", what, B, M, (long long)N, U, H, K);
  int bits = 1;
  while (bits < 31 && (1 << bits) < K) ++bits;              // bits(K - 1), at least 1
  if (M > SID_EXCL_MAX_M || H > RQB_MAX_LEVELS || H * bits > 62) {
    rqb_set_error("%s: need M <= %d, H <= %d and H * bits(K - 1) <= 62 (M = %d, H = %d, K = %d)", what, SID_EXCL_MAX_M,
                  RQB_MAX_LEVELS, M, H, K);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(items && start && (inv || N == 0) && (leaf_key || U == 0) && pos && keys && count, "%s: null pointer", what);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long* lk = reinterpret_cast<const long long*>(leaf_key);
  long long* kk = reinterpret_cast<long long*>(keys);
  auto kernel = include ? (M <= SID_EXCL_THREADS       ? sid_filter_kernel<1, true>
                           : M <= 2 * SID_EXCL_THREADS ? sid_filter_kernel<2, true>
                           : M <= 4 * SID_EXCL_THREADS ? sid_filter_kernel<4, true>
                                                       : sid_filter_kernel<8, true>)
                        : (M <= SID_EXCL_THREADS       ? sid_filter_kernel<1, false>
                           : M <= 2 * SID_EXCL_THREADS ? sid_filter_kernel<2, false>
                           : M <= 4 * SID_EXCL_THREADS ? sid_filter_kernel<4, false>
                                                       : sid_filter_kernel<8, false>);
  kernel<<<B, SID_EXCL_THREADS, 0, st>>>(items, M, N, inv, start, lk, U, H, K, pos, kk, count, ex);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_sid_exclusion_build(const int64_t* items, int B, int M, int64_t N, const int* inv, const int* start,
                                          const int64_t* leaf_key, int U, int H, int K, int* pos, int64_t* blocked, int* count,
                                          void* stream) {
  return sid_filter_build(items, B, M, N, inv, start, leaf_key, U, H, K, pos, blocked, count, SidExcl{}, false,
                          "sid_exclusion_build", stream);
}

extern "C" int rqb200_sid_inclusion_build(const int64_t* items, int B, int M, int64_t N, const int* inv, const int* start,
                                          const int64_t* leaf_key, int U, int H, int K, int* pos, int64_t* keys, int* count,
                                          const int* ex_pos, const int64_t* ex_blocked, const int* ex_count, int ex_M, int ex_H,
                                          void* stream) {
  SidExcl ex;
  const int rc = sid_excl_of(ex_pos, ex_blocked, ex_count, ex_M, ex_H, 0, "sid_inclusion_build", ex);
  if (rc != RQB_OK) return rc;
  return sid_filter_build(items, B, M, N, inv, start, leaf_key, U, H, K, pos, keys, count, ex, true, "sid_inclusion_build", stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// Rank histogram of evaluate/metrics.py's TopKAccumulator: row b's rank is its first candidate whose D columns all equal
// actual[b] (`.all(-1).max(-1)`), k when none does; hist[rank] += 1.  Integer atomics: the sums do not depend on their order.
// item_mode: a value -1 (a padded or unresolvable item) never matches.
__global__ void sid_topk_rank_hist_kernel(const int64_t* __restrict__ actual, int64_t a_stride, const int64_t* __restrict__ cand,
                                          int64_t c_stride, int B, int k, int D, int item_mode, unsigned long long* __restrict__ hist) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
    const int64_t* a = actual + (int64_t)b * a_stride;
    const int64_t* c = cand + (int64_t)b * c_stride;
    int rank = k;
    for (int j = 0; j < k && rank == k; ++j) {
      bool match = true;
      for (int d = 0; d < D && match; ++d) {
        const int64_t v = a[d];
        match = c[(int64_t)j * D + d] == v && !(item_mode && v == -1);
      }
      if (match) rank = j;
    }
    atomicAdd(hist + rank, 1ull);
  }
}

extern "C" int rqb200_sid_topk_rank_hist(const int64_t* actual, int64_t a_stride, const int64_t* cand, int64_t c_stride, int B, int k,
                                         int D, int item_mode, int64_t* hist, void* stream) {
  RQB_CHECK_ARG(B >= 0 && k > 0 && D > 0 && a_stride >= D && c_stride >= (int64_t)k * D,
                "sid_topk_rank_hist: bad argument (B = %d, k = %d, D = %d)", B, k, D);
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(actual && cand && hist, "sid_topk_rank_hist: null pointer");
  int grid = (B + 255) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  sid_topk_rank_hist_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      actual, a_stride, cand, c_stride, B, k, D, item_mode, reinterpret_cast<unsigned long long*>(hist));
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// The same histogram from exact ranks (rank_items' target_rank): hist[rank] += 1 for rank in [0, k), hist[k] += 1 otherwise.
__global__ void sid_rank_hist_kernel(const int64_t* __restrict__ rank, int B, int64_t k, unsigned long long* __restrict__ hist) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
    const int64_t r = rank[b];
    atomicAdd(hist + ((r >= 0 && r < k) ? r : k), 1ull);
  }
}

extern "C" int rqb200_sid_rank_hist(const int64_t* rank, int B, int64_t k, int64_t* hist, void* stream) {
  RQB_CHECK_ARG(B >= 0 && k > 0, "sid_rank_hist: bad argument (B = %d, k = %lld)", B, (long long)k);
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(rank && hist, "sid_rank_hist: null pointer");
  int grid = (B + 255) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  sid_rank_hist_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(rank, B, k,
                                                                                reinterpret_cast<unsigned long long*>(hist));
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Wide levels of both searches: up to 1024 beams per history, where sid_beam_topk_kernel (kp <= 32, k <= 32) and
// sid_sample_select_kernel (kp * nc <= 1024, k <= 32) stop.  One thread-block cluster of 1, 2, 4 or 8 CTAs per history, one
// launch per level.  CTA r of the cluster owns a contiguous range of the history's beams: it computes their log-sum-exps
// (exhaustive) or their nc-sample draws (sampled, sid_warp_top_n), builds their child masks (sid_beam_mask<FILTER>) and forms
// its candidates' keys
//   v(e) = sid_topk_key(score) << 21 | (2^21 - 1 - e),   e = beam * K + code (exhaustive) or beam * nc + j (sampled),
// distinct within a history (E <= 1024 * 2048 = 2^21), so "the k largest keys" is exactly the narrow kernels' order: descending
// score (-0 folded into +0), equal scores by ascending e.  The scores are those of the narrow kernels, with the same explicit
// roundings, so both give the same bits wherever both run.
// Selection is a radix selection over the cluster (8-bit digits, stopping once the chosen bin holds exactly the entries still
// wanted): each CTA histograms its own candidates, reads its peers' histograms through distributed shared memory after one
// cluster barrier per pass and decides the same digit redundantly.  The histograms are double-buffered: the buffer a pass
// clears was last read by the peers before they reached this pass's barrier.  The kept keys are then gathered into CTA 0,
// sorted descending there (cub::BlockRadixSort, at most 1024 of them) and written out.  Histograms are integer counts and the
// final sort orders distinct keys, so no result depends on the cluster size or on the order of atomics.
// A CTA keeps its 32-bit score keys in shared memory while its slice holds at most SID_WIDE_SMEM_KEYS of them.  Above that
// the exhaustive kernel recomputes them from the logits on every pass (bit-identical, as sid_beam_topk_kernel<false>), and the
// sampled kernel re-reads them from its global workspace, where every draw is kept.
#define SID_WIDE_MAX_BEAMS 1024
#define SID_WIDE_MAX_NC 64
#define SID_WIDE_MAX_SEL 1024                               // kept keys (k <= 1024)
#define SID_WIDE_SMEM_KEYS (16 * 1024)                      // score keys per CTA held in shared memory
#define SID_WIDE_E_BITS 21
#define SID_WIDE_TOPK_THREADS 512
#define SID_WIDE_SAMPLE_THREADS 256
#define SID_WIDE_MAX_CLUSTER 8

struct SidWideShared {
  int hist[2][256];                                         // this CTA's histogram, double-buffered across passes
  int ctl[3];                                               // chosen digit, entries above its bin, entries in its bin
  unsigned int nsel;                                        // CTA 0: kept keys gathered so far
  unsigned long long sel[SID_WIDE_MAX_SEL];                 // CTA 0: the kept keys
};

template <int NT>
using SidWideSort = cub::BlockRadixSort<unsigned long long, NT, SID_WIDE_MAX_SEL / NT>;

__device__ __forceinline__ unsigned long long sid_wide_key(unsigned int key, int e) {
  return ((unsigned long long)key << SID_WIDE_E_BITS) | (unsigned int)((1 << SID_WIDE_E_BITS) - 1 - e);
}

__device__ __forceinline__ float sid_topk_key_inverse(unsigned int key) {
  return __uint_as_float((key & 0x80000000u) ? key ^ 0x80000000u : ~key);
}

// Every CTA of the cluster (cs CTAs, one history): the `want` largest keys v(e) of the history, e over this CTA's candidates
// [e0, e1) with key_at(e) their 32-bit score keys.  On return CTA 0 holds them in s.sel[0, want), in no particular order.
// Starts and ends with cluster barriers between which no CTA touches a peer's shared memory before the peer has initialised it.
template <typename KeyAt>
__device__ void sid_wide_select(const KeyAt& key_at, int e0, int e1, int want, int cs, SidWideShared& s) {
  const int nt = blockDim.x, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned int lt = (1u << lane) - 1u;
  unsigned long long prefix = 0, pmask = 0;
  int pass = 0;
  for (int shift = 48; shift >= 0; shift -= 8, ++pass) {    // v has 21 + 32 = 53 bits
    int* hist = s.hist[pass & 1];
    for (int base = e0; base < e1; base += nt) {
      const int e = base + threadIdx.x;
      int d = 256;
      if (e < e1) {
        const unsigned long long v = sid_wide_key(key_at(e), e);
        if ((v & pmask) == prefix) d = (int)((v >> shift) & 255u);
      }
      const unsigned int same = __match_any_sync(0xffffffffu, d);
      if (d < 256 && (same & lt) == 0) atomicAdd(&hist[d], __popc(same));   // one add per distinct digit of the warp
    }
    cluster_sync_all();                                     // every CTA's histogram of this pass is complete
    if (w == 0) {
      int c[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) c[j] = 0;
      for (int r = 0; r < cs; ++r) {                        // the cluster's bins lane * 8 .. lane * 8 + 7, peers in rank order
        const uint32_t a = cluster_map(smem_u32(hist + lane * 8), (uint32_t)r);
#pragma unroll
        for (int j = 0; j < 8; ++j) c[j] += ld_shared_cluster_s32(a + 4 * j);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += c[j];
      int suf = sum;                                        // entries in bins >= lane * 8
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
            s.ctl[0] = lane * 8 + j;
            s.ctl[1] = acc;
            s.ctl[2] = c[j];
            break;
          }
          acc += c[j];
        }
      }
    } else {                                                // the next pass's buffer: the peers read it before this barrier
      int* next = s.hist[(pass + 1) & 1];
      for (int i = threadIdx.x - 32; i < 256; i += nt - 32) next[i] = 0;
    }
    __syncthreads();
    want -= s.ctl[1];
    prefix |= (unsigned long long)s.ctl[0] << shift;
    pmask |= 255ull << shift;
    if (s.ctl[2] == want) break;                            // the whole bin is kept: the threshold is decided
  }
  // the kept set: keys whose decided digits are above the prefix or equal to it, appended to CTA 0's list
  const uint32_t nsel0 = cluster_map(smem_u32(&s.nsel), 0), sel0 = cluster_map(smem_u32(s.sel), 0);
  for (int base = e0; base < e1; base += nt) {
    const int e = base + threadIdx.x;
    unsigned long long v = 0;
    bool keep = false;
    if (e < e1) {
      v = sid_wide_key(key_at(e), e);
      keep = (v & pmask) >= prefix;
    }
    const unsigned int bk = __ballot_sync(0xffffffffu, keep);
    if (bk == 0) continue;
    uint32_t at = 0;
    if (lane == 0) at = atom_add_shared_cluster_u32(nsel0, (uint32_t)__popc(bk));
    at = __shfl_sync(0xffffffffu, at, 0);
    if (keep) st_shared_cluster_u64(sel0 + 8u * (at + (uint32_t)__popc(bk & lt)), v);
  }
  cluster_sync_all();                                       // CTA 0 holds every kept key
}

// CTA 0 after sid_wide_select: keys[i] = the kept key of rank threadIdx.x * IPT + i (descending; 0 past the n kept)
template <int NT>
__device__ __forceinline__ void sid_wide_sort(SidWideShared& s, typename SidWideSort<NT>::TempStorage& tmp, int n,
                                              unsigned long long (&keys)[SID_WIDE_MAX_SEL / NT]) {
  constexpr int IPT = SID_WIDE_MAX_SEL / NT;
#pragma unroll
  for (int i = 0; i < IPT; ++i) {
    const int r = threadIdx.x * IPT + i;
    keys[i] = r < n ? s.sel[r] : 0ull;                      // every real key is above 0: sid_topk_key(-inf) > 0
  }
  SidWideSort<NT>(tmp).SortDescending(keys, 0, 32 + SID_WIDE_E_BITS);
}

__device__ __forceinline__ void sid_wide_init(SidWideShared& s) {
  for (int i = threadIdx.x; i < 512; i += blockDim.x) (&s.hist[0][0])[i] = 0;
  if (threadIdx.x == 0) s.nsel = 0;
}

// The exhaustive level (sid_beam_topk_kernel's scores) for history blockIdx.x / cs; this CTA owns beams
// [rank * per_cta, rank * per_cta + per_cta) of the history.
template <bool KEYS_IN_SMEM, int FILTER>
__global__ void __launch_bounds__(SID_WIDE_TOPK_THREADS, 2) sid_beam_topk_wide_kernel(
    const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ generated, const float* __restrict__ log_probas,
    int kp, int h, int k, int K, int cs, int per_cta, SidTrie trie, int64_t* __restrict__ out_generated,
    float* __restrict__ out_log_probas, int64_t* __restrict__ out_parent, int* __restrict__ bad, SidExcl ex) {
  constexpr int NT = SID_WIDE_TOPK_THREADS, IPT = SID_WIDE_MAX_SEL / NT;
  extern __shared__ __align__(16) unsigned char sid_smem[];
  __shared__ SidWideShared s;
  __shared__ typename SidWideSort<NT>::TempStorage sort_tmp;
  const int W = NT >> 5, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = (int)cluster_ctarank(), b = blockIdx.x / cs, KW = (K + 31) >> 5;
  const int beam0 = min(kp, rank * per_cta), nb = min(kp, beam0 + per_cta) - beam0;
  const int64_t row0 = (int64_t)b * kp;
  float* s_lse = reinterpret_cast<float*>(sid_smem);                             // [per_cta]
  float* s_plp = s_lse + per_cta;                                                // [per_cta]
  unsigned int* s_mask = reinterpret_cast<unsigned int*>(s_plp + per_cta);       // [per_cta][KW]
  unsigned int* s_key = s_mask + (size_t)per_cta * KW;                           // [per_cta * K] when KEYS_IN_SMEM
  sid_wide_init(s);
  for (int i = w; i < nb; i += W) {                         // warp per beam: row maximum, then log-sum-exp (as the narrow kernel)
    const float* x = logits + (row0 + beam0 + i) * ld;
    float m = -INFINITY;
    bool odd = false;
    for (int c = lane; c < K; c += 32) {
      const float v = x[c];
      m = fmaxf(m, v);
      odd |= v != v || v == INFINITY;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    odd = __any_sync(0xffffffffu, odd);
    float sum = 0.f;
    for (int c = lane; c < K; c += 32) sum += expf(x[c] - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) {
      s_lse[i] = m + logf(sum);
      s_plp[i] = log_probas ? log_probas[row0 + beam0 + i] : 0.f;
      if (bad && (odd || m == -INFINITY)) atomicAdd(bad, 1);
    }
    sid_beam_mask<FILTER>(trie, ex, b, generated + (row0 + beam0 + i) * h, h, K, s_mask + (size_t)i * KW, lane);
  }
  __syncthreads();
  const int e0 = beam0 * K, e1 = (beam0 + nb) * K;
  auto score_key = [=](int e) -> unsigned int {
    const int beam = e / K, c = e - beam * K, i = beam - beam0;
    const float lp = __fadd_rn(__fsub_rn(logits[(row0 + beam) * ld + c], s_lse[i]), s_plp[i]);
    const float sc = sid_extension_score(sid_mask_has(s_mask + (size_t)i * KW, c), lp);
    return sid_topk_key(sc == 0.f ? 0.f : sc);
  };
  if (KEYS_IN_SMEM) {
    for (int e = e0 + threadIdx.x; e < e1; e += NT) s_key[e - e0] = score_key(e);
    __syncthreads();
    sid_wide_select([=](int e) { return s_key[e - e0]; }, e0, e1, k, cs, s);
  } else {
    sid_wide_select(score_key, e0, e1, k, cs, s);
  }
  if (rank != 0) return;
  unsigned long long keys[IPT];
  sid_wide_sort<NT>(s, sort_tmp, k, keys);
#pragma unroll
  for (int i = 0; i < IPT; ++i) {
    const int r = threadIdx.x * IPT + i;
    if (r >= k) continue;
    const int e = (1 << SID_WIDE_E_BITS) - 1 - (int)(keys[i] & ((1u << SID_WIDE_E_BITS) - 1));
    const int beam = e / K;
    const int64_t o = (int64_t)b * k + r;
    out_log_probas[o] = sid_topk_key_inverse((unsigned int)(keys[i] >> SID_WIDE_E_BITS));
    out_parent[o] = row0 + beam;
    int64_t* g = out_generated + o * (h + 1);
    for (int j = 0; j < h; ++j) g[j] = generated[(row0 + beam) * h + j];
    g[h] = e - beam * K;
  }
}

// The sampled level (sid_sample_select_kernel's draws and scores) for history blockIdx.x / cs.  Each of the CTA's warps draws
// one beam at a time into its own buffers; every draw's token goes to ws_tok [B][kp * nc] and its score key to shared memory
// (KEYS_IN_SMEM) or ws_key [B][kp * nc].  WARP: the warped draw from the head's logits, as sid_sample_select_kernel's.
template <bool KEYS_IN_SMEM, int FILTER, bool WARP>
__global__ void __launch_bounds__(SID_WIDE_SAMPLE_THREADS, WARP ? 1 : 0) sid_sample_select_wide_kernel(
    const float* __restrict__ probas, int64_t p_stride, const float* __restrict__ noise, int64_t n_stride,
    const int64_t* __restrict__ generated, const float* __restrict__ log_probas, int kp, int nc, int h, int k, int K, int cs,
    int per_cta, SidTrie trie, int64_t* __restrict__ out_generated, float* __restrict__ out_log_probas,
    int64_t* __restrict__ out_parent, int64_t* __restrict__ samples, float* __restrict__ samp_log_p, int* __restrict__ reject,
    int* __restrict__ ws_tok, unsigned int* __restrict__ ws_key, SidExcl ex, float temp, double top_p) {
  constexpr int NT = SID_WIDE_SAMPLE_THREADS, IPT = SID_WIDE_MAX_SEL / NT, W = NT >> 5;
  extern __shared__ __align__(16) unsigned char sid_smem[];
  __shared__ SidWideShared s;
  __shared__ typename SidWideSort<NT>::TempStorage sort_tmp;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = (int)cluster_ctarank(), b = blockIdx.x / cs, KW = (K + 31) >> 5, E = kp * nc;
  const int beam0 = min(kp, rank * per_cta), nb = min(kp, beam0 + per_cta) - beam0;
  int64_t* s_tok = reinterpret_cast<int64_t*>(sid_smem) + (size_t)w * nc;                                  // [W][nc]
  unsigned int* s_rkey = reinterpret_cast<unsigned int*>(reinterpret_cast<int64_t*>(sid_smem) + (size_t)W * nc);   // [W][K]
  int* s_hist = reinterpret_cast<int*>(s_rkey + (size_t)W * K) + w * 256;   // [W][256], 8-byte aligned (W nc 8 + W K 4 bytes in)
  unsigned int* s_sk = reinterpret_cast<unsigned int*>(s_hist - w * 256 + W * 256) + w * nc;               // [W][nc]
  int* s_si = reinterpret_cast<int*>(s_sk - w * nc + W * nc) + w * nc;                                     // [W][nc]
  unsigned int* s_mask = reinterpret_cast<unsigned int*>(s_si - w * nc + W * nc) + w * KW;                 // [W][KW]
  unsigned int* s_key = s_mask - w * KW + W * KW;                                                          // [per_cta * nc]
  s_rkey += (size_t)w * K;
  int* tok_b = ws_tok + (int64_t)b * E;
  sid_wide_init(s);
  for (int i = w; i < nb; i += W) {
    const int beam = beam0 + i;
    const int64_t row = (int64_t)b * kp + beam;
    const float* p = probas + row * p_stride;
    const float* q = noise + row * n_stride;
    float lse = 0.f;
    if (WARP) {
      const SidWarpedRow wr = sid_warped_keys(p, q, K, temp, top_p, s_rkey, reinterpret_cast<unsigned long long*>(s_hist), lane);
      lse = wr.lse;
      if (reject && lane == 0 && wr.bad) atomicAdd(reject, 1);
    } else {
      bool bad = false, nonzero = false;
      for (int c = lane; c < K; c += 32) {
        const float pv = p[c];
        bad |= !(pv >= 0.f) || pv == INFINITY;
        nonzero |= pv != 0.f;
        s_rkey[c] = sid_topk_key(__fdiv_rn(pv, q[c]));
      }
      bad = __any_sync(0xffffffffu, bad);
      nonzero = __any_sync(0xffffffffu, nonzero);
      if (reject && lane == 0 && (bad || !nonzero)) atomicAdd(&reject[bad ? 0 : 1], 1);
    }
    __syncwarp();
    sid_warp_top_n(s_rkey, K, nc, s_hist, s_sk, s_si, s_tok, lane);
    sid_beam_mask<FILTER>(trie, ex, b, generated + row * h, h, K, s_mask, lane);
    const float plp = log_probas ? log_probas[row] : 0.f;
    for (int r = lane; r < nc; r += 32) {
      const int64_t tok = s_tok[r];
      float lp, sc;
      if (WARP) {
        const bool drawn = s_rkey[tok] != 0u;
        lp = drawn ? __fsub_rn(p[tok], lse) : -INFINITY;
        if (samples) samples[row * nc + r] = tok;
        if (samp_log_p) samp_log_p[row * nc + r] = lp;
        sc = sid_extension_score(drawn && sid_mask_has(s_mask, (int)tok), __fadd_rn(lp, plp));
      } else {
        lp = logf(p[tok]);
        if (samples) samples[row * nc + r] = tok;
        if (samp_log_p) samp_log_p[row * nc + r] = lp;
        sc = sid_extension_score(sid_mask_has(s_mask, (int)tok), lp + plp);
      }
      const unsigned int key = sid_topk_key(sc == 0.f ? 0.f : sc);
      const int e = beam * nc + r;
      tok_b[e] = (int)tok;
      if (KEYS_IN_SMEM) s_key[e - beam0 * nc] = key;
      else ws_key[(int64_t)b * E + e] = key;
    }
    __syncwarp();
  }
  __syncthreads();
  const int e0 = beam0 * nc, e1 = (beam0 + nb) * nc, n = min(k, E);
  if (KEYS_IN_SMEM) sid_wide_select([=](int e) { return s_key[e - e0]; }, e0, e1, n, cs, s);
  else sid_wide_select([=](int e) { return ws_key[(int64_t)b * E + e]; }, e0, e1, n, cs, s);
  if (rank != 0) return;
  unsigned long long keys[IPT];
  sid_wide_sort<NT>(s, sort_tmp, n, keys);
#pragma unroll
  for (int i = 0; i < IPT; ++i) {
    const int r = threadIdx.x * IPT + i;
    if (r >= k) continue;
    int e = 0;                                              // k > kp * nc: the remaining slots repeat entry 0 with -inf
    float lp = -INFINITY;
    if (r < n) {
      e = (1 << SID_WIDE_E_BITS) - 1 - (int)(keys[i] & ((1u << SID_WIDE_E_BITS) - 1));
      lp = sid_topk_key_inverse((unsigned int)(keys[i] >> SID_WIDE_E_BITS));
    }
    const int beam = e / nc;
    const int64_t o = (int64_t)b * k + r, parent = (int64_t)b * kp + beam;
    out_log_probas[o] = lp;
    out_parent[o] = parent;
    int64_t* g = out_generated + o * (h + 1);
    for (int j = 0; j < h; ++j) g[j] = generated[parent * h + j];
    g[h] = tok_b[e];
  }
}

// A wide kernel instance for cluster size cs: the function, its dynamic shared memory and its beams per CTA
struct SidWideLaunch {
  const void* fn;
  size_t smem;
  int per_cta;
};

// Picks the cluster size (forced: 1, 2, 4 or 8; 0: choose) of a wide launch over B histories of kp beams, `work` elements read
// per history, and sets up cfg (grid B * cs) for it.  pick(cs) gives the instance for cs.  The choice spreads small batches
// over the GPU (B * cs up to the SM count, at least 16 K elements per CTA) and takes the nearest size whose shared memory fits
// and of which a cluster can be resident (cudaOccupancyMaxActiveClusters).
template <typename Pick>
static int sid_wide_plan(int B, int kp, int64_t work, int forced, int nt, const Pick& pick, cudaStream_t st, const char* what,
                         cudaLaunchConfig_t& cfg, cudaLaunchAttribute& attr, SidWideLaunch& L, int& cs) {
  int dev = 0, nsm = 0, optin = 0;
  RQB_CUDA(cudaGetDevice(&dev));
  RQB_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  RQB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  if (forced != 0 && forced != 1 && forced != 2 && forced != 4 && forced != 8) {
    rqb_set_error("%s: cluster = %d (0 to choose, or 1, 2, 4 or 8)", what, forced);
    return RQB_ERR_INVALID;
  }
  int pref = 1;
  while (pref < SID_WIDE_MAX_CLUSTER && 2 * pref <= kp && (int64_t)B * pref < nsm && work / (2 * pref) >= 16 * 1024) pref *= 2;
  int order[SID_WIDE_MAX_CLUSTER], n = 0;
  if (forced) {
    order[n++] = forced;
  } else {
    for (int c = pref; c >= 1; c /= 2) order[n++] = c;
    for (int c = 2 * pref; c <= SID_WIDE_MAX_CLUSTER; c *= 2) order[n++] = c;
  }
  attr.id = cudaLaunchAttributeClusterDimension;
  cfg = cudaLaunchConfig_t{};
  cfg.blockDim = dim3(nt);
  cfg.stream = st;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  for (int i = 0; i < n; ++i) {
    const int c = order[i];
    const SidWideLaunch l = pick(c);
    cudaFuncAttributes fa;
    RQB_CUDA(cudaFuncGetAttributes(&fa, l.fn));
    if (fa.sharedSizeBytes + l.smem > (size_t)optin) continue;
    RQB_CUDA(cudaFuncSetAttribute(l.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)l.smem));
    attr.val.clusterDim.x = c;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.gridDim = dim3((unsigned)(B * c));
    cfg.dynamicSmemBytes = l.smem;
    int active = 0;
    if (cudaOccupancyMaxActiveClusters(&active, l.fn, &cfg) != cudaSuccess) {
      cudaGetLastError();
      active = 0;
    }
    if (active > 0) {
      L = l;
      cs = c;
      return RQB_OK;
    }
  }
  rqb_set_error("%s: no cluster size %s fits kp = %d beams of this level in shared memory", what,
                forced ? "of the one asked for" : "of 1, 2, 4 or 8", kp);
  return RQB_ERR_UNSUPPORTED;
}

template <int FILTER>
static SidWideLaunch sid_beam_topk_wide_pick(int kp, int K, int cs) {
  const int per_cta = (kp + cs - 1) / cs;
  const bool keys = (int64_t)per_cta * K <= SID_WIDE_SMEM_KEYS;
  const size_t smem = (size_t)per_cta * (2 * sizeof(float) + ((K + 31) / 32) * sizeof(unsigned int)) +
                      (keys ? (size_t)per_cta * K * sizeof(unsigned int) : 0);
  return {keys ? (const void*)sid_beam_topk_wide_kernel<true, FILTER> : (const void*)sid_beam_topk_wide_kernel<false, FILTER>,
          smem, per_cta};
}

template <int FILTER>
static int sid_beam_topk_wide_launch(const float* logits, int64_t logits_stride, const int64_t* generated, const float* log_probas,
                                     int B, int kp, int h, int k, int K, const SidTrie& trie, int64_t* out_generated,
                                     float* out_log_probas, int64_t* out_parent, int* bad, const SidExcl& ex, int cluster,
                                     cudaStream_t st) {
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr;
  SidWideLaunch L;
  int cs = 0;
  const int rc = sid_wide_plan(B, kp, (int64_t)kp * K, cluster, SID_WIDE_TOPK_THREADS,
                               [&](int c) { return sid_beam_topk_wide_pick<FILTER>(kp, K, c); }, st, "sid_trie_beam_topk_wide",
                               cfg, attr, L, cs);
  if (rc != RQB_OK) return rc;
  SidTrie tr = trie;
  SidExcl fx = ex;
  void* args[] = {&logits, &logits_stride, &generated, &log_probas, &kp, &h, &k, &K, &cs, &L.per_cta, &tr,
                  &out_generated, &out_log_probas, &out_parent, &bad, &fx};
  RQB_CUDA(cudaLaunchKernelExC(&cfg, L.fn, args));
  return RQB_OK;
}

static int sid_beam_topk_wide(const float* logits, int64_t logits_stride, const int64_t* generated, const float* log_probas, int B,
                              int kp, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
                              float* out_log_probas, int64_t* out_parent, int* bad, const SidExcl& ex, int cluster, void* stream) {
  RQB_CHECK_ARG(B >= 0 && kp > 0 && h >= 0 && h < C && C <= 8 && k > 0 && K > 0 && logits_stride >= K,
                "sid_trie_beam_topk_wide: bad argument (B=%d kp=%d h=%d k=%d C=%d K=%d)", B, kp, h, k, C, K);
  if (K > SID_TOPK_MAX_K || k > SID_WIDE_MAX_SEL || k > K || kp > SID_WIDE_MAX_BEAMS) {
    rqb_set_error("sid_trie_beam_topk_wide: need K <= %d, k <= %d, k <= K, kp <= %d (K = %d, k = %d, kp = %d)", SID_TOPK_MAX_K,
                  SID_WIDE_MAX_SEL, SID_WIDE_MAX_BEAMS, K, k, kp);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(logits && prefix_workspace && out_generated && out_log_probas && out_parent && (h == 0 || generated) &&
                    (h == 0 || log_probas), "sid_trie_beam_topk_wide: null pointer");
  const SidTrie trie{reinterpret_cast<const unsigned char*>(prefix_workspace), h + 1};
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (sid_filter_mode(ex)) {
    case SID_FILTER_INCLUDE:
      return sid_beam_topk_wide_launch<SID_FILTER_INCLUDE>(logits, logits_stride, generated, log_probas, B, kp, h, k, K, trie,
                                                           out_generated, out_log_probas, out_parent, bad, ex, cluster, st);
    case SID_FILTER_EXCLUDE:
      return sid_beam_topk_wide_launch<SID_FILTER_EXCLUDE>(logits, logits_stride, generated, log_probas, B, kp, h, k, K, trie,
                                                           out_generated, out_log_probas, out_parent, bad, ex, cluster, st);
    default:
      return sid_beam_topk_wide_launch<SID_FILTER_NONE>(logits, logits_stride, generated, log_probas, B, kp, h, k, K, trie,
                                                        out_generated, out_log_probas, out_parent, bad, ex, cluster, st);
  }
}

extern "C" int rqb200_sid_trie_beam_topk_wide(const float* logits, int64_t logits_stride, const int64_t* generated,
                                              const float* log_probas, int B, int kp, int h, int k, int C, int K,
                                              const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                              int64_t* out_parent, int* bad, int cluster, void* stream) {
  return sid_beam_topk_wide(logits, logits_stride, generated, log_probas, B, kp, h, k, C, K, prefix_workspace, out_generated,
                            out_log_probas, out_parent, bad, SidExcl{}, cluster, stream);
}

extern "C" int rqb200_sid_trie_beam_topk_wide_excluding(const float* logits, int64_t logits_stride, const int64_t* generated,
                                                        const float* log_probas, int B, int kp, int h, int k, int C, int K,
                                                        const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                                        int64_t* out_parent, int* bad, int cluster, const int* ex_pos,
                                                        const int64_t* ex_blocked, const int* ex_count, int ex_M, int ex_H,
                                                        void* stream) {
  SidExcl ex;
  const int rc = sid_excl_of(ex_pos, ex_blocked, ex_count, ex_M, ex_H, h + 1, "sid_trie_beam_topk_wide_excluding", ex);
  if (rc != RQB_OK) return rc;
  return sid_beam_topk_wide(logits, logits_stride, generated, log_probas, B, kp, h, k, C, K, prefix_workspace, out_generated,
                            out_log_probas, out_parent, bad, ex, cluster, stream);
}

extern "C" int rqb200_sid_trie_beam_topk_wide_including(const float* logits, int64_t logits_stride, const int64_t* generated,
                                                        const float* log_probas, int B, int kp, int h, int k, int C, int K,
                                                        const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                                        int64_t* out_parent, int* bad, int cluster, const int* in_pos,
                                                        const int64_t* in_keys, const int* in_count, int in_M, int in_H,
                                                        void* stream) {
  SidExcl in;
  const int rc = sid_excl_of(in_pos, in_keys, in_count, in_M, in_H, h + 1, "sid_trie_beam_topk_wide_including", in, true);
  if (rc != RQB_OK) return rc;
  return sid_beam_topk_wide(logits, logits_stride, generated, log_probas, B, kp, h, k, C, K, prefix_workspace, out_generated,
                            out_log_probas, out_parent, bad, in, cluster, stream);
}

extern "C" size_t rqb200_sid_trie_sample_select_wide_workspace_bytes(int B, int kp, int nc) {
  return B < 0 || kp < 0 || nc < 0 ? 0 : (size_t)B * kp * nc * (sizeof(int) + sizeof(unsigned int));
}

template <int FILTER, bool WARP>
static SidWideLaunch sid_sample_select_wide_pick(int kp, int nc, int K, int cs) {
  constexpr int W = SID_WIDE_SAMPLE_THREADS / 32;
  const int per_cta = (kp + cs - 1) / cs;
  const bool keys = (int64_t)per_cta * nc <= SID_WIDE_SMEM_KEYS;
  const size_t smem = (size_t)W * (nc * sizeof(int64_t) + (K + 256 + 2 * nc + (K + 31) / 32) * 4) +
                      (keys ? (size_t)per_cta * nc * sizeof(unsigned int) : 0);
  return {keys ? (const void*)sid_sample_select_wide_kernel<true, FILTER, WARP>
               : (const void*)sid_sample_select_wide_kernel<false, FILTER, WARP>,
          smem, per_cta};
}

template <int FILTER, bool WARP>
static int sid_sample_select_wide_launch(const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride,
                                         const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k,
                                         int K, const SidTrie& trie, int64_t* out_generated, float* out_log_probas,
                                         int64_t* out_parent, int64_t* samples, float* samp_log_p, int* reject, int* ws_tok,
                                         unsigned int* ws_key, const SidExcl& ex, int cluster, float temp, float top_p,
                                         cudaStream_t st) {
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr;
  SidWideLaunch L;
  int cs = 0;
  const int rc = sid_wide_plan(B, kp, (int64_t)kp * K, cluster, SID_WIDE_SAMPLE_THREADS,
                               [&](int c) { return sid_sample_select_wide_pick<FILTER, WARP>(kp, nc, K, c); }, st,
                               "sid_trie_sample_select_wide", cfg, attr, L, cs);
  if (rc != RQB_OK) return rc;
  SidTrie tr = trie;
  SidExcl fx = ex;
  double mass = top_p;                                      // the kernel's nucleus mass parameter
  void* args[] = {&probas, &probas_stride, &noise, &noise_stride, &generated, &log_probas, &kp, &nc, &h, &k, &K, &cs, &L.per_cta,
                  &tr, &out_generated, &out_log_probas, &out_parent, &samples, &samp_log_p, &reject, &ws_tok, &ws_key, &fx,
                  &temp, &mass};
  RQB_CUDA(cudaLaunchKernelExC(&cfg, L.fn, args));
  return RQB_OK;
}

template <bool WARP>
static int sid_sample_select_wide(const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride,
                                  const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K,
                                  const void* prefix_workspace, int64_t* out_generated, float* out_log_probas, int64_t* out_parent,
                                  int64_t* samples, float* samp_log_p, int* reject, void* workspace, size_t workspace_bytes,
                                  int cluster, const SidExcl& ex, float temp, float top_p, void* stream) {
  RQB_CHECK_ARG(B >= 0 && kp > 0 && nc > 0 && h >= 0 && h < C && C <= 8 && k > 0 && K > 0 && probas_stride >= K &&
                    noise_stride >= K, "sid_trie_sample_select_wide: bad argument (B=%d kp=%d nc=%d h=%d k=%d C=%d K=%d)", B, kp,
                nc, h, k, C, K);
  if (WARP && sid_check_warp(temp, top_p, "sid_trie_sample_select_warped_wide") != RQB_OK) return RQB_ERR_INVALID;
  if (nc > K || K > SID_SAMPLE_MAX_K || nc > SID_WIDE_MAX_NC || kp > SID_WIDE_MAX_BEAMS || k > SID_WIDE_MAX_SEL) {
    rqb_set_error("sid_trie_sample_select_wide: need nc <= K <= %d, nc <= %d, kp <= %d, k <= %d (nc = %d, K = %d, kp = %d, k = %d)",
                  SID_SAMPLE_MAX_K, SID_WIDE_MAX_NC, SID_WIDE_MAX_BEAMS, SID_WIDE_MAX_SEL, nc, K, kp, k);
    return RQB_ERR_UNSUPPORTED;
  }
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(probas && noise && prefix_workspace && out_generated && out_log_probas && out_parent && workspace &&
                    (h == 0 || generated) && (h == 0 || log_probas), "sid_trie_sample_select_wide: null pointer");
  if (workspace_bytes < rqb200_sid_trie_sample_select_wide_workspace_bytes(B, kp, nc)) {
    rqb_set_error("sid_trie_sample_select_wide: workspace too small");
    return RQB_ERR_WORKSPACE;
  }
  int* ws_tok = reinterpret_cast<int*>(workspace);
  unsigned int* ws_key = reinterpret_cast<unsigned int*>(ws_tok + (size_t)B * kp * nc);
  const SidTrie trie{reinterpret_cast<const unsigned char*>(prefix_workspace), h + 1};
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (sid_filter_mode(ex)) {
    case SID_FILTER_INCLUDE:
      return sid_sample_select_wide_launch<SID_FILTER_INCLUDE, WARP>(probas, probas_stride, noise, noise_stride, generated, log_probas, B,
                                                               kp, nc, h, k, K, trie, out_generated, out_log_probas, out_parent,
                                                               samples, samp_log_p, reject, ws_tok, ws_key, ex, cluster, temp, top_p, st);
    case SID_FILTER_EXCLUDE:
      return sid_sample_select_wide_launch<SID_FILTER_EXCLUDE, WARP>(probas, probas_stride, noise, noise_stride, generated, log_probas, B,
                                                               kp, nc, h, k, K, trie, out_generated, out_log_probas, out_parent,
                                                               samples, samp_log_p, reject, ws_tok, ws_key, ex, cluster, temp, top_p, st);
    default:
      return sid_sample_select_wide_launch<SID_FILTER_NONE, WARP>(probas, probas_stride, noise, noise_stride, generated, log_probas, B,
                                                            kp, nc, h, k, K, trie, out_generated, out_log_probas, out_parent,
                                                            samples, samp_log_p, reject, ws_tok, ws_key, ex, cluster, temp, top_p, st);
  }
}

extern "C" int rqb200_sid_trie_sample_select_wide(const float* probas, int64_t probas_stride, const float* noise,
                                                  int64_t noise_stride, const int64_t* generated, const float* log_probas, int B,
                                                  int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace,
                                                  int64_t* out_generated, float* out_log_probas, int64_t* out_parent,
                                                  int64_t* samples, float* samp_log_p, int* reject, void* workspace,
                                                  size_t workspace_bytes, int cluster, void* stream) {
  return sid_sample_select_wide<false>(probas, probas_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                       prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, reject,
                                       workspace, workspace_bytes, cluster, SidExcl{}, 1.f, 1.f, stream);
}

extern "C" int rqb200_sid_trie_sample_select_wide_excluding(
    const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* reject, void* workspace,
    size_t workspace_bytes, int cluster, const int* ex_pos, const int64_t* ex_blocked, const int* ex_count, int ex_M, int ex_H,
    void* stream) {
  SidExcl ex;
  const int rc = sid_excl_of(ex_pos, ex_blocked, ex_count, ex_M, ex_H, h + 1, "sid_trie_sample_select_wide_excluding", ex);
  if (rc != RQB_OK) return rc;
  return sid_sample_select_wide<false>(probas, probas_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                       prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, reject,
                                       workspace, workspace_bytes, cluster, ex, 1.f, 1.f, stream);
}

extern "C" int rqb200_sid_trie_sample_select_wide_including(
    const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* reject, void* workspace,
    size_t workspace_bytes, int cluster, const int* in_pos, const int64_t* in_keys, const int* in_count, int in_M, int in_H,
    void* stream) {
  SidExcl in;
  const int rc = sid_excl_of(in_pos, in_keys, in_count, in_M, in_H, h + 1, "sid_trie_sample_select_wide_including", in, true);
  if (rc != RQB_OK) return rc;
  return sid_sample_select_wide<false>(probas, probas_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                       prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, reject,
                                       workspace, workspace_bytes, cluster, in, 1.f, 1.f, stream);
}

extern "C" int rqb200_sid_trie_sample_select_warped_wide(const float* logits, int64_t logits_stride, const float* noise,
                                                         int64_t noise_stride, const int64_t* generated, const float* log_probas,
                                                         int B, int kp, int nc, int h, int k, int C, int K,
                                                         const void* prefix_workspace, int64_t* out_generated,
                                                         float* out_log_probas, int64_t* out_parent, int64_t* samples,
                                                         float* samp_log_p, int* bad, void* workspace, size_t workspace_bytes,
                                                         int cluster, float temperature, float top_p, void* stream) {
  return sid_sample_select_wide<true>(logits, logits_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                      prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, bad, workspace,
                                      workspace_bytes, cluster, SidExcl{}, temperature, top_p, stream);
}

extern "C" int rqb200_sid_trie_sample_select_warped_wide_excluding(
    const float* logits, int64_t logits_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* bad, void* workspace,
    size_t workspace_bytes, int cluster, float temperature, float top_p, const int* ex_pos, const int64_t* ex_blocked,
    const int* ex_count, int ex_M, int ex_H, void* stream) {
  SidExcl ex;
  const int rc = sid_excl_of(ex_pos, ex_blocked, ex_count, ex_M, ex_H, h + 1, "sid_trie_sample_select_warped_wide_excluding", ex);
  if (rc != RQB_OK) return rc;
  return sid_sample_select_wide<true>(logits, logits_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                      prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, bad, workspace,
                                      workspace_bytes, cluster, ex, temperature, top_p, stream);
}

extern "C" int rqb200_sid_trie_sample_select_warped_wide_including(
    const float* logits, int64_t logits_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* bad, void* workspace,
    size_t workspace_bytes, int cluster, float temperature, float top_p, const int* in_pos, const int64_t* in_keys,
    const int* in_count, int in_M, int in_H, void* stream) {
  SidExcl in;
  const int rc = sid_excl_of(in_pos, in_keys, in_count, in_M, in_H, h + 1, "sid_trie_sample_select_warped_wide_including", in,
                             true);
  if (rc != RQB_OK) return rc;
  return sid_sample_select_wide<true>(logits, logits_stride, noise, noise_stride, generated, log_probas, B, kp, nc, h, k, C, K,
                                      prefix_workspace, out_generated, out_log_probas, out_parent, samples, samp_log_p, bad, workspace,
                                      workspace_bytes, cluster, in, temperature, top_p, stream);
}
