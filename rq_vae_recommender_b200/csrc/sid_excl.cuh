// Per-history item filters of the semantic-id search, item retrieval and exact ranking: exclusion sets
// (rqb200_sid_exclusion_build in csrc/sid.cu writes them; the search kernels of sid.cu and t5rank_select_kernel of t5rank.cu read
// them) and allow-lists (rqb200_sid_inclusion_build; the search and retrieval kernels of sid.cu read them).  Both have one layout.
//
// For history b of B, with M entries per history and H levels:
//   pos[b][0 .. n)          exclusion: the distinct excluded items, inclusion: the eligible items (allowed, retrievable and not
//                           excluded), as positions in the item table's sorted row array, ascending (n = count[b][0]); the table's
//                           order is lexicographic, so the items under one trie prefix are one run of them;
//   keys[b][l - 1][0 .. m)  the packed keys (level 0 most significant, K-ary) of l-prefixes, ascending (m = count[b][l],
//                           l = 1..H): exclusion, the blocked prefixes (every retrievable item under them is excluded); inclusion,
//                           the valid prefixes (at least one eligible item under them);
//   count[b][H + 1]         the entries outside [-1, N) (counted, otherwise ignored).
// A null count pointer means "no filter": every consumer then runs its code without it.  A consumer takes one filter: an
// inclusion has the exclusion folded in.
#pragma once
#include <cstdint>

#define SID_EXCL_MAX_M 4096

// the compile-time filter mode of a consumer kernel
enum SidFilterMode { SID_FILTER_NONE = 0, SID_FILTER_EXCLUDE = 1, SID_FILTER_INCLUDE = 2 };

struct SidExcl {
  const int* pos;
  const long long* keys;
  const int* count;
  int M, H;
  bool include;                                             // an allow-list (rqb200_sid_inclusion_build), else an exclusion set
  __device__ __forceinline__ bool on() const { return count != nullptr; }
  __device__ __forceinline__ const int* pos_of(int64_t b) const { return pos + b * M; }
  __device__ __forceinline__ int npos(int64_t b) const { return __ldg(count + b * (H + 2)); }
  __device__ __forceinline__ const long long* keys_of(int64_t b, int l) const { return keys + (b * H + (l - 1)) * M; }
  __device__ __forceinline__ int nkeys(int64_t b, int l) const { return __ldg(count + b * (H + 2) + l); }
};

// first i in [0, n) with a[i] >= v (n when none)
template <typename T>
__device__ __forceinline__ int sid_lower_bound(const T* a, int n, T v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// excluded positions (ascending xp[0, nx)) inside [s, e)
__device__ __forceinline__ int sid_excluded_in(const int* xp, int nx, int s, int e) {
  return sid_lower_bound(xp, nx, e) - sid_lower_bound(xp, nx, s);
}

// the d-th (0-based) position at or after s that is not excluded.  With j excluded positions below it, it is s + d + j; the
// excluded x_i >= s lie below it exactly when the kept positions before x_i, x_i - s - i, are at most d (nondecreasing in i).
__device__ __forceinline__ int sid_nth_kept(const int* xp, int nx, int s, int d) {
  const int a = sid_lower_bound(xp, nx, s);
  int lo = 0, hi = nx - a;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (xp[a + mid] - mid - s > d) hi = mid;
    else lo = mid + 1;
  }
  return s + d + lo;
}
