// Tensor-core tokeniser for sm_90a: wgmma fp16 candidate filter + exact fp32 re-rank, K = 256 m codes per level (m = 1..8).
//
// Result contract: identical to rqb200_rq_forward(mode = EVAL, ids only) -- the hard-argmin chain of
// modules/quantize.py:113-128,159-161 x L + modules/rqvae.py:125-132 (what semids.py:125 consumes).
//
//   S_l[b,k]  = fp16(x_b) . fp16(c_{l,k})            (wgmma m64n256k16, fp32 accumulate in registers)
//   h_l[b,k]  = T_l[b,k] - S_l[b,k] / 2^s,  T = cc/2 + sum_{j<l} G_{jl}[id_j(b), k]   (G = float64 Gram tables rounded once: every
//               level is scored from the ONE fp16 image of x, which stays in shared memory for all L levels)
//   candidates(b) = { k : h <= min_k h + 2 eps_b }    eps_b = DETERMINISTIC bound on |h - exact half-distance| (tc_eps, tc_common.cuh)
//   one candidate -> it is the exact argmin;  else the candidates are re-scored with the exact fp32 arithmetic of the
//   CUDA-core kernel (sequential fp32 residual, (xx + cc) - 2 dot, first index wins ties).
//
// One CTA per SM, persistent over 64-row tiles, three warpgroups with their own register budgets (setmaxnreg):
//   WG0, warps 0-3   MMA and scoring: per level and 256-code block, 4 x wgmma per 64-wide k chunk into a 64 x 256 register
//     (scorer)       accumulator, then score.  All 256 codes of a block sit in one thread quad, so the block minimum and its
//                    candidate bits are quad shuffles; a row with one candidate takes it, rows with more go to a shared queue.
//                    It never converts and never re-ranks.
//   WG1, warps 4-7   convert the next tile's rows from their x stages to the fp16 image (K-major SWIZZLE_128B, resident for
//     (helper)       all levels of a tile) and measure ||fp16(x) - x||^2 and ||x||^2 per row; re-rank the queued rows of each
//                    level exactly, any warp taking the next queued row.
//   WG2, warp 8      producer of one 32 KB stage ring (bulk copies counted on an mbarrier per stage).  Per tile it first
//                    stages the tile's fp32 rows, 128 columns per stage (one tensor copy of the 64 x 128 box), then for
//                    every (level, block, k chunk) the prepared 16 KB blocks of codes [256 cb, 256 cb + 128) and
//                    [256 cb + 128, 256 cb + 256).  Only its lane 0 issues copies; warps 9-11 exit at once.  The helper
//                    consumes the x stages and the scorer the codebook stages; each walks the same stage counter and skips
//                    the other's stages.
//
// Hand-offs of tile t, on four mbarriers that every thread of the signalling warpgroup arrives on:
//   scorer  waits IMG_FULL(t); per level l: MMA(l) (after the last level's MMAs complete it arrives on IMG_FREE(t)), waits
//           RR_DONE of the level before (for l = 0: level L-1 of tile t-1), scores and selects, arrives on Q_READY(l).
//   helper  waits IMG_FREE(t-1) and converts tile t, keeping the row statistics in registers; waits Q_READY(L-1) of tile t-1
//           (the scorer no longer reads rowinfo), writes rowinfo, arrives on IMG_FULL(t); re-ranks level L-1 of tile t-1 and
//           arrives on RR_DONE; then for l = 0 .. L-2 waits Q_READY(l), re-ranks level l of tile t, arrives on RR_DONE.
// So the scorer writes the ids, candidate words and queue of a level only once the previous level's re-rank has drained
// them, and the helper writes the image and rowinfo only once the scorer is done with them: none of them is doubled, and the
// shared memory is the single-warpgroup layout's plus four mbarriers.  Each barrier's waiter is never more than one phase
// behind (every arrival needs the other side's previous wait), so parity waits are exact.  The ring cannot deadlock at any
// depth: the producer issues a tile's x stages after the previous tile's last codebook stage, and the helper consumes them
// only after IMG_FREE, which needs nothing but earlier stages.  Each level's re-rank runs under the next level's MMAs, the
// conversion under the last level's scoring.
//
// Two kernels share every stage but the candidate selection:
//   rq_tcx_kernel          K = 256: one accumulator holds the whole level, so the row minimum and the candidate words stay in
//                          registers and only the queued rows store their words.  Ids are 8-bit.
//   rq_tcx_blocked_kernel  K = 512 .. 2048: a level is scored one 256-code BLOCK at a time.  Block cb keeps the codes with
//                          h <= M_cb + 2 eps, M_cb = the running row minimum over blocks 0..cb; M_cb >= the final minimum M, so
//                          every block keeps a superset of its share of the final candidate set.  At the end of the level every
//                          block whose minimum is above M + 2 eps is dropped whole: a row whose final candidate set is one code
//                          ends with exactly that code, so the re-rank rate is the unblocked filter's (tests/tc_blocked_model.py).
//                          Candidate words of every row go to shared memory and ids are 16-bit.
// One kernel with a runtime block loop for every K was 2-4 % slower at K = 256 on the H100, even specialised by template.
#include <cuda.h>
#include <cudaTypedefs.h>

#include "tc_common.cuh"
#include "wgmma.cuh"

#define TX_R 64                                   // rows per tile = wgmma M
#define TX_NB_MAX 4                               // ring stages
#define TX_STAGE_BYTES (2 * TC_BSTAGE_BYTES)      // 256 codes x 64 k fp16 = 32 KB = 64 rows x 128 columns of fp32 x
#define TX_XCOLS 128                              // columns of x per stage: a 512-byte row
#define TX_XROW_BYTES (TX_XCOLS * 4)
#define TX_XGROUP 8                               // rows a converter warp reads from a stage at once
#define TX_SLOT_BYTES (TX_R * TC_KC * 2)          // one k chunk of the x image: 8 KB
#define TX_THREADS 384                            // scorer, helper and producer warpgroups
#define TX_REG_LAUNCH 168                         // registers per thread at launch: 65536 / 384, rounded down to 8
#define TX_REG_SCORER 240                         // setmaxnreg of each role: the scorer raises, the others lower
#define TX_REG_HELPER 160
#define TX_REG_PRODUCER 40
static_assert(TX_REG_LAUNCH * TX_THREADS <= 65536 && TX_REG_SCORER >= TX_REG_LAUNCH && TX_REG_HELPER <= TX_REG_LAUNCH &&
                  TX_REG_PRODUCER <= TX_REG_LAUNCH && TX_REG_SCORER + TX_REG_HELPER + TX_REG_PRODUCER <= 3 * TX_REG_LAUNCH,
              "setmaxnreg budgets must fit the registers the CTA is launched with");
#define TX_SMEM_LIMIT 232448                      // 227 KB of opt-in shared memory per block

struct TxSmem {
  uint64_t full[TX_NB_MAX], empty[TX_NB_MAX];
  uint64_t img_full, img_free;                    // the image of a tile written (helper) / last read (scorer)
  uint64_t q_ready, rr_done;                      // a level's queue complete (scorer) / its re-rank done (helper)
  uint32_t fl_count, fl_next;                     // queue of rows that need the exact re-rank
  uint32_t rowinfo[TX_R];                         // bf16_up(||fp16(x)-x||^2) << 16 | bf16_up(||x||^2)
  unsigned char flist[TX_R];
};

struct TxParams {
  CUtensorMap xmap;              // x as a [B][D] fp32 tensor (row pitch ldx), boxes of TX_R rows x TX_XCOLS columns
  const float* x;
  int64_t ldx;
  int B, D, K, L, nkc, nblk, ntiles, nb;
  const TcHeader* hdr;
  const float* cc;               // [L][K]  fp32 cc of the exact kernels
  const float* hcc;              // [L][K]  cc / 2 from float64
  const float* gram;             // [L(L-1)/2][K][K]
  const float* cbf;              // [L][K][D] fp32 codebook copy (exact re-rank)
  const unsigned char* blob;     // [L][K/128][nkc][16 KB] fp16 codebook images
  int64_t* ids;                  // [B][L]
  int* stats;                    // optional: [0] rows re-ranked, [1] candidates re-scored, [2] rows with >= 3 candidates
};

// Dynamic shared memory of a CTA, in order (tcx_smem_bytes sizes it):
//   x image [nkc][8 KB] | ring [nb][32 KB] (x rows or codebook blocks) | TxSmem |
//   cmask [TX_R][K / 32]   candidate bits (code 32 w + b -> word w, bit b): of the queued rows at K = 256, of every row above
//   bmin  [TX_R][K / 256]  K > 256 only: per-block minimum, NaN if the block holds a NaN score
//   ids   [L][TX_R]        ids of the tile: Id = uint8_t at K = 256 (16-bit ids would cost a ring stage at D = 768, L = 8),
//                          uint16_t above
template <class Id> struct TxShared {
  unsigned char* sC;
  TxSmem* ms;
  uint32_t* cmask;
  float* bmin;
  Id* ids;
};
template <class Id> __device__ __forceinline__ TxShared<Id> tx_shared(unsigned char* tsm, const TxParams& p, int K) {
  const int nblk = K / TC_K;
  TxShared<Id> sh;
  sh.sC = tsm + p.nkc * TX_SLOT_BYTES;
  sh.ms = reinterpret_cast<TxSmem*>(sh.sC + p.nb * TX_STAGE_BYTES);
  sh.cmask = reinterpret_cast<uint32_t*>(sh.ms + 1);
  sh.bmin = reinterpret_cast<float*>(sh.cmask + TX_R * (K / 32));
  sh.ids = reinterpret_cast<Id*>(sh.bmin + (nblk > 1 ? TX_R * nblk : 0));
  return sh;
}
static size_t tcx_smem_bytes(int D, int K, int L, int nb) {
  const int nblk = K / TC_K;
  return (size_t)(D / TC_KC) * TX_SLOT_BYTES + (size_t)nb * TX_STAGE_BYTES + sizeof(TxSmem) + (size_t)TX_R * (K / 32) * 4 +
         (nblk > 1 ? (size_t)TX_R * nblk * 4 + (size_t)L * TX_R * 2 : (size_t)L * TX_R);
}

// candidate margin of a row at a level: 2 eps (1 + 2^-16) from the published statistics
__device__ __forceinline__ float tx_margin(const TcLevelConst& lc, uint32_t ri) {
  return 2.f * tc_eps(lc, __uint_as_float(ri & 0xffff0000u), __uint_as_float(ri << 16)) * 1.0000153f;
}
__device__ __forceinline__ void tx_helper_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }   // the helper's 4 warps
template <uint32_t N> __device__ __forceinline__ void tx_reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N> __device__ __forceinline__ void tx_reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
__device__ __forceinline__ float tx_min_nan(float a, float b) {       // NaN if either is NaN
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// ring and hand-off barriers and an empty re-rank queue, visible to all warps on return
__device__ __forceinline__ void tx_init(unsigned char* tsm, TxSmem* ms) {
  if (threadIdx.x == 0) {
    if ((smem_u32(tsm) & 1023u) != 0) __trap();              // the swizzle pattern needs a 1024-byte aligned base
    for (int i = 0; i < TX_NB_MAX; ++i) { mbar_init(&ms->full[i], 1); mbar_init(&ms->empty[i], 4); }
    mbar_init(&ms->img_full, 128); mbar_init(&ms->img_free, 128);
    mbar_init(&ms->q_ready, 128); mbar_init(&ms->rr_done, 128);
    ms->fl_count = 0; ms->fl_next = 0;
    fence_mbar_init();
  }
  __syncthreads();
}

// producer (lane 0 of warp 8): per tile, its x stages (the helper's), then (level, block, k chunk) (the scorer's).  It
// waits for a free slot and arms its mbarrier with the stage's byte count.  X stage c is ONE tensor copy of the box of rows
// [row0, row0 + 64) and columns [128 c, 128 c + 128): 512 bytes per row, with zeros past B and past D (when D % 128 == 64)
// that the converter never reads; the copy counts the whole box.  One copy per stage rather than 64 bulk copies of a
// 512-byte row each: the step is 14-18 % shorter on the H100 (README).  A codebook stage is two 16 KB bulk copies.
__device__ __forceinline__ void tx_produce(const TxParams& p, unsigned char* sC, TxSmem* ms, int nblk) {
  const int nkc = p.nkc, nxs = (p.D + TX_XCOLS - 1) / TX_XCOLS;
  const uint32_t nb = (uint32_t)p.nb;
  uint32_t s = 0;
  for (int unit = blockIdx.x; unit < p.ntiles; unit += gridDim.x) {
    const int row0 = unit * TX_R;
    for (int c = 0; c < nxs; ++c, ++s) {
      const uint32_t st = s % nb, u = s / nb;
      mbar_wait_guarded(&ms->empty[st], (u & 1) ^ 1, 1);
      mbar_expect_tx(&ms->full[st], TX_STAGE_BYTES);
      tensor_g2s_2d(sC + st * TX_STAGE_BYTES, &p.xmap, c * TX_XCOLS, row0, &ms->full[st]);
    }
    for (int l = 0; l < p.L; ++l)
      for (int cb = 0; cb < nblk; ++cb)
        for (int kc = 0; kc < nkc; ++kc, ++s) {
          const uint32_t st = s % nb, u = s / nb;
          mbar_wait_guarded(&ms->empty[st], (u & 1) ^ 1, 1);
          mbar_expect_tx(&ms->full[st], TX_STAGE_BYTES);
          unsigned char* dst = sC + st * TX_STAGE_BYTES;
          const size_t h0 = (size_t)(l * nblk + cb) * 2;
          bulk_g2s(dst, p.blob + (h0 * nkc + kc) * TC_BSTAGE_BYTES, TC_BSTAGE_BYTES, &ms->full[st]);
          bulk_g2s(dst + TC_BSTAGE_BYTES, p.blob + ((h0 + 1) * nkc + kc) * TC_BSTAGE_BYTES, TC_BSTAGE_BYTES, &ms->full[st]);
        }
  }
}

// fp16 image + row statistics of the tile at row0 from its x stages, the next ones of the ring (s counts the stages
// consumed): helper warp w converts rows [16w, 16w + 16); lane = float4 column of every 512-byte stage row.  Each warp
// releases a stage once its rows are read.  The per-lane sums of a row run over the columns in order, so the statistics do
// not depend on the stage width.  Rows past B are zeros and are never read.  Returns, in lane i < 16, the rowinfo word of
// row 16w + i; the caller publishes it and makes the image visible to the tensor core.
__device__ __forceinline__ uint32_t tx_convert(const TxParams& p, TxSmem* ms, uint32_t x_base, const unsigned char* sC, int row0,
                                               uint32_t& s) {
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, lane4 = lane * 4, D = p.D;
  const int nxs = (D + TX_XCOLS - 1) / TX_XCOLS, nr = min(16, p.B - row0 - warp * 16);   // rows of this warp below B
  const uint32_t nb = (uint32_t)p.nb;
  float s2[16], e2[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) { s2[i] = 0.f; e2[i] = 0.f; }
#pragma unroll 1
  for (int c4 = 0; c4 < nxs; ++c4, ++s) {
    const uint32_t st = s % nb;
    const int c = c4 * TX_XCOLS + lane4;
    mbar_wait_guarded(&ms->full[st], (s / nb) & 1, 2);
    const float4* srcp = reinterpret_cast<const float4*>(sC + st * TX_STAGE_BYTES + warp * 16 * TX_XROW_BYTES) + lane;
    // TX_XGROUP rows at a time.  The image stores below carry no memory clobber, so the compiler may issue a group's stage
    // loads ahead of the previous group's stores (they never overlap); the stage wait and release above and below are
    // compiler barriers either way
#pragma unroll
    for (int i0 = 0; i0 < 16; i0 += TX_XGROUP) {
      float4 v[TX_XGROUP];
#pragma unroll
      for (int j = 0; j < TX_XGROUP; ++j) {
        v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i0 + j < nr && c < D) v[j] = srcp[(i0 + j) * (TX_XROW_BYTES / 16)];
      }
      if (c >= D) continue;
#pragma unroll
      for (int j = 0; j < TX_XGROUP; ++j) {
        const int i = i0 + j, R = warp * 16 + i;
        const float4 a = v[j];
        const __half2 h0 = __floats2half2_rn(a.x, a.y), h1 = __floats2half2_rn(a.z, a.w);
        // the MEASURED rounding error of this row: fp16(x) - x is exact in fp32 (nearby values, or a flush to zero / inf)
        const float2 b0 = __half22float2(h0), b1 = __half22float2(h1);
        const float d0 = b0.x - a.x, d1 = b0.y - a.y, d2 = b1.x - a.z, d3 = b1.y - a.w;
        s2[i] = fmaf(a.x, a.x, fmaf(a.y, a.y, fmaf(a.z, a.z, fmaf(a.w, a.w, s2[i]))));
        e2[i] = fmaf(d0, d0, fmaf(d1, d1, fmaf(d2, d2, fmaf(d3, d3, e2[i]))));
        const uint32_t addr = x_base + (uint32_t)(c >> 6) * TX_SLOT_BYTES + (uint32_t)R * 128u +
                              ((((uint32_t)(c & 63) >> 3) ^ ((uint32_t)R & 7u)) << 4) + (uint32_t)(c & 7) * 2u;
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(*reinterpret_cast<const uint32_t*>(&h0)),
                     "r"(*reinterpret_cast<const uint32_t*>(&h1)));
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&ms->empty[st]);
  }
  uint32_t ri = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float a = warp_sum(s2[i]), b = warp_sum(e2[i]);
    if (lane == i) ri = (tc_bf16_up(b) << 16) | tc_bf16_up(a);
  }
  return ri;
}

// S = X . C^T of one 256-code block over the next nkc ring stages (s counts the stages consumed); a stage is released as
// soon as the MMAs that read it have completed
__device__ __forceinline__ void tx_mma(float (&acc)[128], TxSmem* ms, uint32_t x_base, uint32_t c_base, int nkc, uint32_t nb,
                                       uint32_t& s) {
  const int lane = threadIdx.x & 31;
  uint32_t prev = 0;
#pragma unroll 1
  for (int kc = 0; kc < nkc; ++kc, ++s) {
    const uint32_t st = s % nb;
    mbar_wait_guarded(&ms->full[st], (s / nb) & 1, 2);
    const uint64_t ad = wg_desc(x_base + kc * TX_SLOT_BYTES), bd = wg_desc(c_base + st * TX_STAGE_BYTES);
    wg_fence_acc(acc);
    wg_fence();
#pragma unroll
    for (int j = 0; j < TC_KC / 16; ++j) wg_m64n256_f16(acc, ad + 2 * j, bd + 2 * j, (kc | j) != 0);
    wg_commit();
    wg_fence_acc(acc);
    if (kc > 0) {
      wg_wait<1>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&ms->empty[prev]);
    }
    prev = st;
  }
  wg_wait<0>();
  wg_fence_acc(acc);
  __syncwarp();
  if (lane == 0) mbar_arrive(&ms->empty[prev]);
}

// score the block of codes [col, col + 256) of a level of K codes: h = T - S / 2^s in place; columns col + 8 jb + 2 q4 + {0, 1}
// of rows r0 (acc[4 jb + 0..1]) and r1 (acc[4 jb + 2..3]).  GC = column groups per chunk of Gram-row loads: 16 (two chunks)
// in the K = 256 kernel, 1.7 % shorter step on the H100 together with its early level constants; 4 in the blocked
// kernel, which was 8-18 % slower at 16 (bench_large_k.py)
template <int GC, class Id>
__device__ __forceinline__ void tx_score(float (&acc)[128], const TxParams& p, const TcLevelConst& lc, int l, int col, int K,
                                         const Id* ids, int r0, int r1) {
  const int q4 = threadIdx.x & 3;
  const float ninv = -1.f / lc.sc;
  if (l == 0) {
#pragma unroll
    for (int jb = 0; jb < 32; ++jb) {
      const float2 t = __ldg(reinterpret_cast<const float2*>(p.hcc + col + 8 * jb + 2 * q4));
      acc[4 * jb + 0] = fmaf(acc[4 * jb + 0], ninv, t.x); acc[4 * jb + 1] = fmaf(acc[4 * jb + 1], ninv, t.y);
      acc[4 * jb + 2] = fmaf(acc[4 * jb + 2], ninv, t.x); acc[4 * jb + 3] = fmaf(acc[4 * jb + 3], ninv, t.y);
    }
  } else {
    // Gram rows of the previous levels' ids, table (j, l) at gram + (l (l - 1) / 2 + j) K^2, summed in level order.  GC
    // column groups at a time: the loads of one table are independent, so a level costs l round trips to L2 per chunk rather
    // than one per column group and table
    const float* g0 = p.gram + (size_t)(l * (l - 1) / 2) * K * K + 2 * q4 + col;
    const float* a0 = g0 + (size_t)ids[r0] * K;
    const float* a1 = g0 + (size_t)ids[r1] * K;
#pragma unroll
    for (int jc = 0; jc < 32; jc += GC) {
      float2 t0[GC], t1[GC];
#pragma unroll
      for (int i = 0; i < GC; ++i) {
        t0[i] = __ldg(reinterpret_cast<const float2*>(a0 + 8 * (jc + i)));
        t1[i] = __ldg(reinterpret_cast<const float2*>(a1 + 8 * (jc + i)));
      }
#pragma unroll 1
      for (int j = 1; j < l; ++j) {
        const float* b0 = g0 + ((size_t)j * K + ids[j * TX_R + r0]) * K;
        const float* b1 = g0 + ((size_t)j * K + ids[j * TX_R + r1]) * K;
#pragma unroll
        for (int i = 0; i < GC; ++i) {
          const float2 u0 = __ldg(reinterpret_cast<const float2*>(b0 + 8 * (jc + i)));
          const float2 u1 = __ldg(reinterpret_cast<const float2*>(b1 + 8 * (jc + i)));
          t0[i].x += u0.x; t0[i].y += u0.y; t1[i].x += u1.x; t1[i].y += u1.y;
        }
      }
#pragma unroll
      for (int i = 0; i < GC; ++i) {
        const int jb = jc + i;
        acc[4 * jb + 0] = fmaf(acc[4 * jb + 0], ninv, t0[i].x); acc[4 * jb + 1] = fmaf(acc[4 * jb + 1], ninv, t0[i].y);
        acc[4 * jb + 2] = fmaf(acc[4 * jb + 2], ninv, t1[i].x); acc[4 * jb + 3] = fmaf(acc[4 * jb + 3], ninv, t1[i].y);
      }
    }
  }
}

// minimum of rows r0 (m0) and r1 (m1) over the quad's 256 scores, in every lane of the quad
__device__ __forceinline__ void tx_quad_min(const float (&acc)[128], float& m0, float& m1) {
  m0 = INFINITY; m1 = INFINITY;
#pragma unroll
  for (int jb = 0; jb < 32; ++jb) {
    m0 = fminf(m0, fminf(acc[4 * jb + 0], acc[4 * jb + 1]));
    m1 = fminf(m1, fminf(acc[4 * jb + 2], acc[4 * jb + 3]));
  }
#pragma unroll
  for (int o = 1; o < 4; o <<= 1) {
    m0 = fminf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
    m1 = fminf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
  }
}

// candidate word w of the block (codes 32 w .. 32 w + 31) of rows r0 (b0) and r1 (b1), in every lane of the quad; NaN keeps
// the code
__device__ __forceinline__ void tx_cand_word(const float (&acc)[128], int w, float thr0, float thr1, uint32_t& b0, uint32_t& b1) {
  const int q4 = threadIdx.x & 3;
  b0 = 0u; b1 = 0u;
#pragma unroll
  for (int t = 0; t < 4; ++t)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const uint32_t bit = 1u << (8 * t + 2 * q4 + e);
      b0 |= !(acc[4 * (4 * w + t) + e] > thr0) ? bit : 0u;
      b1 |= !(acc[4 * (4 * w + t) + 2 + e] > thr1) ? bit : 0u;
    }
  b0 |= __shfl_xor_sync(0xffffffffu, b0, 1); b0 |= __shfl_xor_sync(0xffffffffu, b0, 2);
  b1 |= __shfl_xor_sync(0xffffffffu, b1, 1); b1 |= __shfl_xor_sync(0xffffffffu, b1, 2);
}

// row r of the tile after the filter: with cnt candidates, the first being `first` (>= K if none).  A row with one candidate
// takes it; any other row in range is queued for the exact re-rank (returns true), a row past B takes a valid code.
template <class Id>
__device__ __forceinline__ bool tx_settle(const TxParams& p, TxSmem* ms, Id* ids, int l, int row0, int r, int cnt, int first,
                                          int K) {
  const int grow = row0 + r;
  if (cnt != 1 && grow < p.B) {
    const uint32_t qi = atomicAdd(&ms->fl_count, 1u);
    ms->flist[qi] = (unsigned char)r;
    return true;
  }
  const int my_id = first >= K ? 0 : first;
  ids[l * TX_R + r] = (Id)my_id;
  if (grow < p.B) p.ids[(int64_t)grow * p.L + l] = my_id;
  return false;
}

// Exact re-rank, by the helper, of the tile's queued rows at level l once the scorer has settled or queued every row
// (Q_READY); any warp takes the next row (same arithmetic as rq_simt.cu: sequential fp32 residual, (xx + cc) - 2 dot,
// candidates in ascending index order with a strict '<': first index wins ties).  Lane covers elements 128 i + 4 lane .. +3
// of a row (6 x LDG.128 per row).  On return every id of the level is in ids[] and the queue is empty again, for the scorer
// once the helper has arrived on RR_DONE.
template <class Id>
__device__ __forceinline__ void tx_rerank(const TxParams& p, const TxShared<Id>& sh, int l, int row0, int K) {
  const int lane = threadIdx.x & 31, lane4 = lane * 4, D = p.D, nw = K / 32;
  TxSmem* const ms = sh.ms;
  const float* ccl = p.cc + (size_t)l * K;
  const float* cl = p.cbf + (size_t)l * K * D;
  const uint32_t nfl = *reinterpret_cast<volatile uint32_t*>(&ms->fl_count);
  int n_rows = 0, n_cand = 0, n_many = 0;
  auto ld_row = [&](const float* base, float4 (&v)[6]) {
#pragma unroll
    for (int i = 0; i < 6; ++i)
      v[i] = (i * 128 + lane4 < D) ? __ldg(reinterpret_cast<const float4*>(base + i * 128 + lane4)) : make_float4(0.f, 0.f, 0.f, 0.f);
  };
#pragma unroll 1
  while (true) {
    uint32_t qi = 0;
    if (lane == 0) qi = atomicAdd(&ms->fl_next, 1u);
    qi = __shfl_sync(0xffffffffu, qi, 0);
    if (qi >= nfl) break;
    const int rrow = ms->flist[qi];
    const int rgrow = row0 + rrow;
    const uint32_t* const cm = sh.cmask + rrow * nw;
    const uint32_t wlo = lane < nw ? cm[lane] : 0u, whi = lane + 32 < nw ? cm[lane + 32] : 0u;   // lane holds words lane, lane + 32
    // first two candidates (ascending code order): their rows, the x row and the first prior code are ALL requested
    // before anything is consumed -- one or two L2 round trips instead of four dependent ones
    uint32_t wcur = 0, mwd = 0;
    int w = 0;
    auto next_cand = [&]() -> int {                         // -1 when the candidate words are exhausted
      while (mwd == 0u) {
        if (w >= nw) return -1;
        mwd = __shfl_sync(0xffffffffu, w < 32 ? wlo : whi, w & 31);
        wcur = (uint32_t)w * 32u;
        ++w;
      }
      const int k = (int)wcur + __ffs(mwd) - 1;
      mwd &= mwd - 1;
      return k;
    };
    int ka = next_cand(), kb = next_cand();
    float4 res[6], va[6], vb[6];
    ld_row(p.x + (int64_t)rgrow * p.ldx, res);
    if (l > 0) ld_row(p.cbf + (size_t)sh.ids[rrow] * D, vb);              // first prior code travels in vb
    if (ka >= 0) ld_row(cl + (size_t)ka * D, va);
#pragma unroll 1
    for (int j = 0; j < l; ++j) {
#pragma unroll
      for (int i = 0; i < 6; ++i) { res[i].x -= vb[i].x; res[i].y -= vb[i].y; res[i].z -= vb[i].z; res[i].w -= vb[i].w; }   // rqvae.py:130, level order
      if (j + 1 < l) ld_row(p.cbf + ((size_t)(j + 1) * K + sh.ids[(j + 1) * TX_R + rrow]) * D, vb);
    }
    if (kb >= 0) ld_row(cl + (size_t)kb * D, vb);
    float cca = (ka >= 0) ? __ldg(ccl + ka) : 0.f, ccb = (kb >= 0) ? __ldg(ccl + kb) : 0.f;
    float best = INFINITY;
    int besti = 0x7fffffff, nc = 0;
    const int firsti = ka;
    float xx = 0.f;
    bool have_xx = false;
#pragma unroll 1
    while (ka >= 0) {
      // per-lane partial sums in the exact kernel's order, then ONE butterfly for all of them
      float da = 0.f, db = 0.f, xp = 0.f;
#pragma unroll
      for (int i = 0; i < 6; ++i) da = tc_dot4(res[i], va[i], da);
      if (kb >= 0) {
#pragma unroll
        for (int i = 0; i < 6; ++i) db = tc_dot4(res[i], vb[i], db);
      }
      if (!have_xx) {
#pragma unroll
        for (int i = 0; i < 6; ++i) xp = tc_dot4(res[i], res[i], xp);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        da += __shfl_xor_sync(0xffffffffu, da, o);
        db += __shfl_xor_sync(0xffffffffu, db, o);
        xp += __shfl_xor_sync(0xffffffffu, xp, o);
      }
      if (!have_xx) { xx = xp; have_xx = true; }
      const float dist_a = (xx + cca) - 2.f * da;           // quantize.py:113-117
      if (dist_a < best) { best = dist_a; besti = ka; }
      ++nc;
      if (kb >= 0) {
        const float dist_b = (xx + ccb) - 2.f * db;
        if (dist_b < best) { best = dist_b; besti = kb; }
        ++nc;
      }
      ka = (kb >= 0) ? next_cand() : -1;
      kb = (ka >= 0) ? next_cand() : -1;
      if (ka >= 0) { ld_row(cl + (size_t)ka * D, va); cca = __ldg(ccl + ka); }
      if (kb >= 0) { ld_row(cl + (size_t)kb * D, vb); ccb = __ldg(ccl + kb); }
    }
    if (besti >= K) besti = firsti < 0 ? 0 : firsti;        // all-NaN distances: keep a valid code
    if (lane == 0) {
      sh.ids[l * TX_R + rrow] = (Id)besti;
      p.ids[(int64_t)rgrow * p.L + l] = besti;
    }
    ++n_rows; n_cand += nc; n_many += (nc >= 3);
  }
  if (p.stats && lane == 0 && n_rows) {
    atomicAdd(p.stats + 0, n_rows);
    atomicAdd(p.stats + 1, n_cand);
    atomicAdd(p.stats + 2, n_many);
  }
  tx_helper_sync();                                         // every id of the level is in ids[]; the queue is drained
  // the reset reaches the scorer with this thread's RR_DONE arrival, and the other helper warps through the scorer's next
  // Q_READY, so no second barrier
  if ((threadIdx.x & 127) == 0) { ms->fl_count = 0; ms->fl_next = 0; }
}

// helper warpgroup: converts each tile into the image and re-ranks its levels, in the hand-off order of the header comment
// (n counts the tiles, so the Q_READY / RR_DONE completion of level l of tile n is the (n L + l)-th)
template <class Id>
__device__ __forceinline__ void tx_helper(const TxParams& p, const TxShared<Id>& sh, uint32_t x_base, int K) {
  TxSmem* const ms = sh.ms;
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const uint32_t L = (uint32_t)p.L, ncs = L * (uint32_t)((K / TC_K) * p.nkc);   // codebook stages of a tile: the scorer's
  uint32_t s = 0, n = 0;
  int prev0 = 0;                                            // row0 of the previous tile
#pragma unroll 1
  for (int unit = blockIdx.x; unit < p.ntiles; unit += gridDim.x, ++n) {
    const int row0 = unit * TX_R;
    if (n > 0) mbar_wait_guarded(&ms->img_free, (n - 1) & 1, 3);
    const uint32_t ri = tx_convert(p, ms, x_base, sh.sC, row0, s);
    s += ncs;
    if (n > 0) mbar_wait_guarded(&ms->q_ready, (n * L - 1) & 1, 4);   // the scorer is done with the last tile's rowinfo
    if (lane < 16) ms->rowinfo[warp * 16 + lane] = ri;
    fence_proxy_async();                                    // generic-proxy image stores -> visible to the tensor core
    mbar_arrive(&ms->img_full);
    if (n > 0) {
      tx_rerank(p, sh, (int)L - 1, prev0, K);
      mbar_arrive(&ms->rr_done);
    }
#pragma unroll 1
    for (uint32_t l = 0; l + 1 < L; ++l) {
      mbar_wait_guarded(&ms->q_ready, (n * L + l) & 1, 4);
      tx_rerank(p, sh, (int)l, row0, K);
      mbar_arrive(&ms->rr_done);
    }
    prev0 = row0;
  }
  if (n > 0) {
    mbar_wait_guarded(&ms->q_ready, (n * L - 1) & 1, 4);
    tx_rerank(p, sh, (int)L - 1, prev0, K);
  }
}

// the helper and producer warpgroups of either kernel, each at its register budget; returns false in the scorer warpgroup,
// which has raised its own
template <class Id>
__device__ __forceinline__ bool tx_side_roles(const TxParams& p, const TxShared<Id>& sh, uint32_t x_base, int K) {
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  if (wg == 2) {
    tx_reg_dec<TX_REG_PRODUCER>();
    if (threadIdx.x == 8 * 32) tx_produce(p, sh.sC, sh.ms, K / TC_K);   // lane 0 of warp 8; the rest have nothing to do
    return true;
  }
  if (wg == 1) {
    tx_reg_dec<TX_REG_HELPER>();
    tx_helper(p, sh, x_base, K);
    return true;
  }
  tx_reg_inc<TX_REG_SCORER>();
  return false;
}

__global__ void __launch_bounds__(TX_THREADS, 1) rq_tcx_kernel(const __grid_constant__ TxParams p) {
  extern __shared__ __align__(1024) unsigned char tsm[];
  const TxShared<uint8_t> sh = tx_shared<uint8_t>(tsm, p, TC_K);
  const uint32_t x_base = smem_u32(tsm), c_base = smem_u32(sh.sC);
  tx_init(tsm, sh.ms);
  if (tx_side_roles(p, sh, x_base, TC_K)) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, q4 = lane & 3;
  const int r0 = warp * 16 + (lane >> 2), r1 = r0 + 8;      // accumulator rows of this thread
  const uint32_t nxs = (uint32_t)((p.D + TX_XCOLS - 1) / TX_XCOLS), L = (uint32_t)p.L;
  uint32_t s = 0, n = 0;
#pragma unroll 1
  for (int unit = blockIdx.x; unit < p.ntiles; unit += gridDim.x, ++n) {
    const int row0 = unit * TX_R;
    s += nxs;                                               // the tile's x stages: the helper's
    mbar_wait_guarded(&sh.ms->img_full, n & 1, 5);
#pragma unroll 1
    for (uint32_t l = 0; l < L; ++l) {
      // the level's constants and the rows' candidate margins before the MMAs, whose wait hides the header's load (rowinfo
      // holds this tile's statistics until the last level's Q_READY)
      const TcLevelConst lc = p.hdr->lv[l];
      const float mg0 = tx_margin(lc, sh.ms->rowinfo[r0]), mg1 = tx_margin(lc, sh.ms->rowinfo[r1]);
      float acc[128];
      tx_mma(acc, sh.ms, x_base, c_base, p.nkc, (uint32_t)p.nb, s);
      if (l + 1 == L) mbar_arrive(&sh.ms->img_free);       // the helper may convert the next tile
      // ids, candidate words and queue of the level before are drained by its re-rank
      if (n | l) mbar_wait_guarded(&sh.ms->rr_done, (n * L + l - 1) & 1, 6);
      tx_score<16>(acc, p, lc, l, 0, TC_K, sh.ids, r0, r1);
      // ---- candidates: the row minimum, then the 8 candidate words in registers; only a queued row stores its words
      float m0, m1;
      tx_quad_min(acc, m0, m1);
      const float thr0 = m0 + mg0, thr1 = m1 + mg1;
      uint32_t w0[8], w1[8];
      int cnt0 = 0, cnt1 = 0, first0 = TC_K, first1 = TC_K;
#pragma unroll
      for (int w = 7; w >= 0; --w) {
        tx_cand_word(acc, w, thr0, thr1, w0[w], w1[w]);
        cnt0 += __popc(w0[w]); cnt1 += __popc(w1[w]);
        first0 = w0[w] ? w * 32 + __ffs(w0[w]) - 1 : first0;
        first1 = w1[w] ? w * 32 + __ffs(w1[w]) - 1 : first1;
      }
      if (q4 < 2) {                                         // lane 4i + 0 finalises row r0, lane 4i + 1 row r1
        const int r = q4 ? r1 : r0;
        if (tx_settle(p, sh.ms, sh.ids, l, row0, r, q4 ? cnt1 : cnt0, q4 ? first1 : first0, TC_K)) {
#pragma unroll
          for (int w = 0; w < 8; ++w) sh.cmask[r * 8 + w] = q4 ? w1[w] : w0[w];
        }
      }
      mbar_arrive(&sh.ms->q_ready);                         // every row of the level is settled or queued
    }
  }
}

__global__ void __launch_bounds__(TX_THREADS, 1) rq_tcx_blocked_kernel(const __grid_constant__ TxParams p) {
  extern __shared__ __align__(1024) unsigned char tsm[];
  const int K = p.K, nblk = p.nblk, nw = K / 32;
  const TxShared<uint16_t> sh = tx_shared<uint16_t>(tsm, p, K);
  const uint32_t x_base = smem_u32(tsm), c_base = smem_u32(sh.sC);
  tx_init(tsm, sh.ms);
  if (tx_side_roles(p, sh, x_base, K)) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, q4 = lane & 3;
  const int r0 = warp * 16 + (lane >> 2), r1 = r0 + 8;      // accumulator rows of this thread
  const uint32_t nxs = (uint32_t)((p.D + TX_XCOLS - 1) / TX_XCOLS), L = (uint32_t)p.L;
  uint32_t s = 0, n = 0;
#pragma unroll 1
  for (int unit = blockIdx.x; unit < p.ntiles; unit += gridDim.x, ++n) {
    const int row0 = unit * TX_R;
    s += nxs;                                               // the tile's x stages: the helper's
    mbar_wait_guarded(&sh.ms->img_full, n & 1, 5);
#pragma unroll 1
    for (uint32_t l = 0; l < L; ++l) {
      float run0 = INFINITY, run1 = INFINITY;                // running row minima over the blocks scored so far
      float thr0 = 0.f, thr1 = 0.f;                          // candidate thresholds of the latest block: the final ones after it
#pragma unroll 1
      for (int cb = 0; cb < nblk; ++cb) {
        float acc[128];
        tx_mma(acc, sh.ms, x_base, c_base, p.nkc, (uint32_t)p.nb, s);
        if (l + 1 == L && cb + 1 == nblk) mbar_arrive(&sh.ms->img_free);   // the helper may convert the next tile
        // ids, candidate words and queue of the level before are drained by its re-rank
        if (cb == 0 && (n | l)) mbar_wait_guarded(&sh.ms->rr_done, (n * L + l - 1) & 1, 6);
        const TcLevelConst lc = p.hdr->lv[l];
        tx_score<4>(acc, p, lc, l, cb * TC_K, K, sh.ids, r0, r1);
        // ---- candidates: the block minimum, the running minimum, then the block's candidate words to shared memory
        float m0, m1;
        tx_quad_min(acc, m0, m1);
        {
          // the block's key for the end-of-level drop: its minimum, NaN when any score is NaN (such a block is never dropped)
          float k0 = m0, k1 = m1;
#pragma unroll
          for (int jb = 0; jb < 32; ++jb) {
            k0 = tx_min_nan(k0, tx_min_nan(acc[4 * jb + 0], acc[4 * jb + 1]));
            k1 = tx_min_nan(k1, tx_min_nan(acc[4 * jb + 2], acc[4 * jb + 3]));
          }
#pragma unroll
          for (int o = 1; o < 4; o <<= 1) {
            k0 = tx_min_nan(k0, __shfl_xor_sync(0xffffffffu, k0, o));
            k1 = tx_min_nan(k1, __shfl_xor_sync(0xffffffffu, k1, o));
          }
          if (q4 == 0) sh.bmin[r0 * nblk + cb] = k0;
          if (q4 == 1) sh.bmin[r1 * nblk + cb] = k1;
        }
        run0 = fminf(run0, m0); run1 = fminf(run1, m1);
        thr0 = run0 + tx_margin(lc, sh.ms->rowinfo[r0]); thr1 = run1 + tx_margin(lc, sh.ms->rowinfo[r1]);
#pragma unroll
        for (int w = 0; w < 8; ++w) {
          uint32_t b0, b1;
          tx_cand_word(acc, w, thr0, thr1, b0, b1);
          if (q4 == 0) sh.cmask[r0 * nw + cb * 8 + w] = b0;  // lane 4i + 0 owns row r0, lane 4i + 1 row r1 (it finalises them below)
          if (q4 == 1) sh.cmask[r1 * nw + cb * 8 + w] = b1;
        }
      }

      if (q4 < 2) {                                         // lane 4i + 0 finalises row r0, lane 4i + 1 row r1
        const int r = q4 ? r1 : r0;
        const float thr = q4 ? thr1 : thr0;
        uint32_t* const cm = sh.cmask + r * nw;
        int cnt = 0, first = K;
#pragma unroll 1
        for (int cb = 0; cb < nblk; ++cb) {
          if (sh.bmin[r * nblk + cb] > thr) {               // no code of this block is within the final margin
#pragma unroll
            for (int w = 0; w < 8; ++w) cm[cb * 8 + w] = 0u;
            continue;
          }
#pragma unroll
          for (int w = 0; w < 8; ++w) {
            const uint32_t b = cm[cb * 8 + w];
            cnt += __popc(b);
            first = (b && first == K) ? (cb * 8 + w) * 32 + __ffs(b) - 1 : first;
          }
        }
        tx_settle(p, sh.ms, sh.ids, l, row0, r, cnt, first, K);
      }
      mbar_arrive(&sh.ms->q_ready);                         // every row of the level is settled or queued
    }
  }
}

// the ring gets as many 32 KB stages (<= TX_NB_MAX) as fit under the 227 KB limit: 4 at K = 256 for every D and L (88 bytes
// to spare at D = 768, L = 8), 3 at K > 256 with D = 768 and at some K > 256 with D = 640 or 704, 4 elsewhere.  tcx_run and
// rqb200_tokenize_tc_ring_stages both take the depth from here.
int tcx_ring_stages(int D, int K, int L) {
  int nbs = TX_NB_MAX;
  while (nbs > 2 && tcx_smem_bytes(D, K, L, nbs) > TX_SMEM_LIMIT) --nbs;
  return nbs;
}

int tcx_run(const float* x, int64_t ldx, int B, const void* state, int D, int K, int L, int64_t* ids, int* stats, int sm_count,
            cudaStream_t st) {
  const char* base = reinterpret_cast<const char*>(state);
  TxParams p{};
  p.x = x; p.ldx = ldx; p.B = B; p.D = D; p.K = K; p.L = L; p.nkc = D / TC_KC; p.nblk = K / TC_K;
  p.ntiles = (B + TX_R - 1) / TX_R;
  p.hdr = reinterpret_cast<const TcHeader*>(base);
  p.cc = reinterpret_cast<const float*>(base + tc_off_cc(K, L));
  p.hcc = reinterpret_cast<const float*>(base + tc_off_hcc(K, L));
  p.gram = reinterpret_cast<const float*>(base + tc_off_gram(K, L));
  p.cbf = reinterpret_cast<const float*>(base + tc_off_cbf(K, L));
  p.blob = reinterpret_cast<const unsigned char*>(base + tc_off_blob(D, K, L));
  p.ids = ids; p.stats = stats;
  p.nb = tcx_ring_stages(D, K, L);
  // the x tensor map: dimension 0 = the D columns (row pitch ldx floats), dimension 1 = the B rows; reads outside it
  // (columns past D, rows past B) fill the box with zeros
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  if (!encode) {
    cudaDriverEntryPointQueryResult q;
    void* fn = nullptr;
    RQB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    if (q != cudaDriverEntryPointSuccess || !fn) {
      rqb_set_error("tokenize_tc_run: the driver has no cuTensorMapEncodeTiled");
      return RQB_ERR_CUDA;
    }
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  const cuuint64_t dims[2] = {(cuuint64_t)D, (cuuint64_t)B}, strides[1] = {(cuuint64_t)ldx * 4u};
  const cuuint32_t box[2] = {TX_XCOLS, TX_R}, estr[2] = {1, 1};
  if (encode(&p.xmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(x), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
    rqb_set_error("tokenize_tc_run: cuTensorMapEncodeTiled failed (B=%d D=%d ldx=%lld)", B, D, (long long)ldx);
    return RQB_ERR_CUDA;
  }
  const size_t smem = tcx_smem_bytes(D, K, L, p.nb);
  // K = 256: one accumulator holds a level; larger K is scored in 256-code blocks
  void (*const kernel)(TxParams) = K == TC_K ? rq_tcx_kernel : rq_tcx_blocked_kernel;
  RQB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = p.ntiles < sm_count ? p.ntiles : sm_count;
  kernel<<<grid, TX_THREADS, smem, st>>>(p);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}
