// Attention-weight dropout of the T5 training passes (csrc/t5enc.cu and csrc/t5dec.cu).  A keep bit is never stored: each is one
// Philox4x32-10 draw keyed on a per-call int64 seed read from device memory and counted by (history, head, query position, key
// position), so a backward derives the same bits as its forward, and the encoder and the decoder draw from one layout.
#pragma once
#include <cstdint>

#include <curand_kernel.h>

// Keep bit of the attention weight of (history b, head n, query position pi, key position pj): one Philox4x32-10 draw, kept when
// its first word is at least thresh = p * 2^32 (so thresh = 0 keeps everything).
__device__ __forceinline__ bool te_keep(uint2 key, int b, int n, int pi, int pj, uint32_t thresh) {
  return curand_Philox4x32_10(make_uint4((unsigned)pj, (unsigned)pi, (unsigned)n, (unsigned)b), key).x >= thresh;
}

__device__ __forceinline__ uint2 te_seed_key(const int64_t* seed) {
  const uint64_t s = (uint64_t)seed[0];
  return make_uint2((unsigned)s, (unsigned)(s >> 32));
}

// 0 <= p < 1 -> the Philox threshold and the kept weights' scale
static inline void dropout_params(float p, uint32_t* thresh, float* scale) {
  *thresh = (uint32_t)((double)p * 4294967296.0);
  *scale = *thresh ? 1.f / (1.f - p) : 1.f;
}
