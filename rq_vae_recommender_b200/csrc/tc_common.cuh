// Shared definitions of the tensor-core tokeniser (csrc/rq_tc.cu: prepare and C ABI; csrc/rq_tcx.cu: the K = 256 and blocked
// kernels): prepared-state layout, filter bound, small device helpers.
// Everything here is static / inline; the result contract is stated at the top of rq_tc.cu.
#pragma once
#include "common.cuh"
#include <cuda_fp16.h>
#include <cmath>
#include <cstdlib>

#define TC_K 256          // codes per block: one wgmma m64n256 accumulator; a level has K = 256 m codes, m = 1..8
#define TC_MAX_K 2048
#define TC_KC 64          // fp16 elements per 128-byte swizzle row
#define TC_MAX_D 768
#define TC_MAX_KC (TC_MAX_D / TC_KC)
#define TC_BSTAGE_BYTES (128 * TC_KC * 2)   // 128 codes x 64 k x fp16 = 16 KB
// Filter error bound: DETERMINISTIC.  With x~ = fp16(x) and
// c~ = fp16(c 2^s) / 2^s,   x~.c~ - x.c = (x~ - x).c~ + x.(c~ - c)   exactly, hence by Cauchy-Schwarz
//   |x~.c~_k - x.c_k| <= ||x~ - x|| ||c~_k|| + ||x|| ||c~_k - c_k||  <=  ex_b chat_l + xn_b ec_l
// ex_b is MEASURED per row by the converter (subnormal flushes and overflow are inside it: an overflowing row gets
// ex = inf and keeps every code), chat_l / ec_l are measured per level by tc_prep_err_kernel.  TC_INFL covers the fp32
// accumulation of those norms and the bf16 round-up of the published row statistics.
#define TC_INFL 1.002f

struct TcLevelConst {
  float sc;      // power-of-two scale applied to the codebook before fp16 conversion
  float chat;    // max_k ||c~_k||_2            (x TC_INFL)
  float ec;      // max_k ||c~_k - c_k||_2      (x TC_INFL)
  float c2max;   // max_k ||c_k||_2
  float gerr;    // roundings of the Gram tables / cc / the score FFMA at this level
  float prior;   // sum_{j<l} c2max_j: bound on the norm of the codes subtracted before this level
  float pad[2];
};

struct TcHeader {
  TcLevelConst lv[RQB_MAX_LEVELS];
  unsigned int amax_bits[RQB_MAX_LEVELS];  // scratch of prepare
  unsigned int chat_bits[RQB_MAX_LEVELS];
  unsigned int ec_bits[RQB_MAX_LEVELS];
  unsigned int c2_bits[RQB_MAX_LEVELS];
};

// eps_b of level l from the published row statistics (ex^2, xn^2): every term is an upper bound, see tests/tc_filter_model.py
__host__ __device__ __forceinline__ float tc_eps(const TcLevelConst& lc, float ex2, float xn2) {
#ifdef __CUDA_ARCH__
  const float ex = __fsqrt_ru(ex2), xn = __fsqrt_ru(xn2);     // rounded UP: every term stays an upper bound; one MUFU each, no slow path
#else
  const float ex = sqrtf(ex2) * 1.0000002f, xn = sqrtf(xn2) * 1.0000002f;
#endif
  const float acc = 7.62939453e-6f * xn * lc.c2max;                                             // 2^-17: tensor-core fp32 accumulation
  const float ref = 7.62939453e-6f * ((xn + lc.prior) * lc.c2max + 0.5f * lc.c2max * lc.c2max); // fp32 noise of the reference's own distances
  return TC_INFL * (ex * lc.chat + xn * lc.ec) + acc + lc.gerr + ref;
}

// Prepared state, in order: header | cc [L][K] | hcc [L][K] | Gram tables [L(L-1)/2][K][K] | codebook pointers |
// fp32 codebooks [L][K][D] | fp16 blob [L][K/128][D/64][16 KB].  The Gram tables dominate at large K (K^2 L(L-1)/2 x 4 bytes:
// 50 MB of the ~80 MB at K = 2048, L = 3, D = 768; 470 MB of the ~0.55 GB at L = 8).
static size_t tc_off_cc(int K, int L) { return rqb_round_up(sizeof(TcHeader), 256); }
static size_t tc_off_hcc(int K, int L) { return tc_off_cc(K, L) + rqb_round_up((size_t)L * K * 4, 256); }
static size_t tc_off_gram(int K, int L) { return tc_off_hcc(K, L) + rqb_round_up((size_t)L * K * 4, 256); }
static size_t tc_off_cbptr(int K, int L) { return tc_off_gram(K, L) + (size_t)(L * (L - 1) / 2) * K * K * 4; }
static size_t tc_off_cbf(int K, int L) { return rqb_round_up(tc_off_cbptr(K, L) + RQB_MAX_LEVELS * 8, 256); }   // fp32 copy [L][K][D]
static size_t tc_off_blob(int D, int K, int L) { return rqb_round_up(tc_off_cbf(K, L) + (size_t)L * K * D * 4, 1024); }
static size_t tc_state_size(int D, int K, int L) { return tc_off_blob(D, K, L) + (size_t)L * (K / 128) * (D / TC_KC) * TC_BSTAGE_BYTES; }

__device__ __forceinline__ uint32_t tc_bf16_up(float v) {   // bf16 bits of the smallest bf16 >= v (v >= 0, inf/nan kept)
  uint32_t b = __float_as_uint(v);
  if ((b & 0x7f800000u) != 0x7f800000u && (b & 0xffffu)) b += 0x10000u;
  return b >> 16;
}

__device__ __forceinline__ float tc_dot4(const float4& a, const float4& b, float acc) {
  return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, fmaf(a.w, b.w, acc))));
}
