// Tensor-core tokeniser for sm_90a: wgmma fp16 candidate filter + exact fp32 re-rank, K = 256 codes per level (one 256-code
// accumulator holds all of a level's codes).  K = 512 .. 2048 is csrc/rq_tcx_blocked.cu.
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
// One CTA per SM, persistent over 64-row tiles:
//   warps 0-3 (one warpgroup)  convert the tile's rows to the fp16 image (K-major SWIZZLE_128B, resident for all levels) and
//                              measure ||fp16(x) - x||^2 and ||x||^2 per row; per level: 4 x wgmma per 64-wide k chunk into a
//                              64 x 256 register accumulator, then score.  All 256 codes of a row sit in one thread quad, so the
//                              row minimum and the candidate set are two quad shuffles; rows with more than one candidate go to
//                              a shared queue that the four warps re-rank exactly.
//   warp 4                     codebook producer: the prepared 16 KB blocks of codes [0,128) and [128,256) of (level, k chunk)
//                              -> one 32 KB stage of a ring (bulk copies counted on an mbarrier); it runs ahead into the next
//                              level and tile while the warpgroup scores and converts.
#include "tc_common.cuh"
#include "wgmma.cuh"

#define TX_R 64                                   // rows per tile = wgmma M
#define TX_NB_MAX 4                               // codebook ring stages
#define TX_STAGE_BYTES (2 * TC_BSTAGE_BYTES)      // 256 codes x 64 k fp16 = 32 KB
#define TX_SLOT_BYTES (TX_R * TC_KC * 2)          // one k chunk of the x image: 8 KB
#define TX_THREADS 160
#define TX_SMEM_LIMIT 232448                      // 227 KB of opt-in shared memory per block

struct TxSmem {
  uint64_t full[TX_NB_MAX], empty[TX_NB_MAX];
  uint32_t fl_count, fl_next;                     // queue of rows that need the exact re-rank
  uint32_t rowinfo[TX_R];                         // bf16_up(||fp16(x)-x||^2) << 16 | bf16_up(||x||^2)
  uint32_t cmask[TX_R][8];                        // candidate bits of the queued rows (code 32 w + b -> word w, bit b)
  unsigned char flist[TX_R];
};

struct TxParams {
  const float* x;
  int64_t ldx;
  int B, D, L, nkc, ntiles, nb;
  const TcHeader* hdr;
  const float* cc;               // [L][256]  fp32 cc of the exact kernels
  const float* hcc;              // [L][256]  cc / 2 from float64
  const float* gram;             // [L(L-1)/2][256][256]
  const float* cbf;              // [L][256][D] fp32 codebook copy (exact re-rank)
  const unsigned char* blob;     // [L][2][nkc][16 KB] fp16 codebook images
  int64_t* ids;                  // [B][L]
  int* stats;                    // optional: [0] rows re-ranked, [1] candidates re-scored, [2] rows with >= 3 candidates
};

// candidate margin of a row at a level: 2 eps (1 + 2^-16) from the published statistics
__device__ __forceinline__ float tx_margin(const TcLevelConst& lc, uint32_t ri) {
  return 2.f * tc_eps(lc, __uint_as_float(ri & 0xffff0000u), __uint_as_float(ri << 16)) * 1.0000153f;
}
__device__ __forceinline__ void tx_wg_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }   // the 4 warps of the warpgroup

__global__ void __launch_bounds__(TX_THREADS, 1) rq_tcx_kernel(const __grid_constant__ TxParams p) {
  extern __shared__ __align__(1024) unsigned char tsm[];
  const int nkc = p.nkc, L = p.L, D = p.D;
  const uint32_t nb = (uint32_t)p.nb;
  unsigned char* sX = tsm;                                   // [nkc][8 KB] fp16 image of the tile's rows
  unsigned char* sC = sX + nkc * TX_SLOT_BYTES;              // [nb][32 KB] codebook ring
  TxSmem* ms = reinterpret_cast<TxSmem*>(sC + nb * TX_STAGE_BYTES);
  unsigned char* const ids8 = reinterpret_cast<unsigned char*>(ms + 1);   // [L][TX_R] ids of the tile
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    if ((smem_u32(tsm) & 1023u) != 0) __trap();              // the swizzle pattern needs a 1024-byte aligned base
    for (int i = 0; i < TX_NB_MAX; ++i) { mbar_init(&ms->full[i], 1); mbar_init(&ms->empty[i], 4); }
    ms->fl_count = 0; ms->fl_next = 0;
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ============================================================== codebook producer
    if (lane == 0) {
      uint32_t s = 0;
      for (int unit = blockIdx.x; unit < p.ntiles; unit += gridDim.x)
        for (int l = 0; l < L; ++l)
          for (int kc = 0; kc < nkc; ++kc, ++s) {
            const uint32_t st = s % nb, u = s / nb;
            mbar_wait_guarded(&ms->empty[st], (u & 1) ^ 1, 1);
            mbar_expect_tx(&ms->full[st], TX_STAGE_BYTES);
            unsigned char* dst = sC + st * TX_STAGE_BYTES;
            bulk_g2s(dst, p.blob + ((size_t)(l * 2) * nkc + kc) * TC_BSTAGE_BYTES, TC_BSTAGE_BYTES, &ms->full[st]);
            bulk_g2s(dst + TC_BSTAGE_BYTES, p.blob + ((size_t)(l * 2 + 1) * nkc + kc) * TC_BSTAGE_BYTES, TC_BSTAGE_BYTES,
                     &ms->full[st]);
          }
    }
    return;
  }

  // ============================================================== warpgroup
  const int q4 = lane & 3;
  const int r0 = warp * 16 + (lane >> 2), r1 = r0 + 8;      // accumulator rows of this thread
  const int lane4 = lane * 4;
  const uint32_t x_base = smem_u32(sX), c_base = smem_u32(sC);
  uint32_t s = 0;
#pragma unroll 1
  for (int unit = blockIdx.x; unit < p.ntiles; unit += gridDim.x) {
    const int row0 = unit * TX_R;
    // ---- fp16 image + row statistics: warp w converts rows [16w, 16w + 16); lane = float4 column of every 512-byte stretch
#pragma unroll 2
    for (int i = 0; i < 16; ++i) {
      const int R = warp * 16 + i, grow = row0 + R;
      const float* xr = p.x + (int64_t)grow * p.ldx;
      float4 v[6];
#pragma unroll
      for (int c4 = 0; c4 < 6; ++c4) {
        const int c = c4 * 128 + lane4;
        v[c4] = (grow < p.B && c < D) ? __ldg(reinterpret_cast<const float4*>(xr + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      float s2 = 0.f, e2 = 0.f;
#pragma unroll
      for (int c4 = 0; c4 < 6; ++c4) {
        const int c = c4 * 128 + lane4;
        if (c < D) {
          const float4 a = v[c4];
          const __half2 h0 = __floats2half2_rn(a.x, a.y), h1 = __floats2half2_rn(a.z, a.w);
          // the MEASURED rounding error of this row: fp16(x) - x is exact in fp32 (nearby values, or a flush to zero / inf)
          const float2 b0 = __half22float2(h0), b1 = __half22float2(h1);
          const float d0 = b0.x - a.x, d1 = b0.y - a.y, d2 = b1.x - a.z, d3 = b1.y - a.w;
          s2 = fmaf(a.x, a.x, fmaf(a.y, a.y, fmaf(a.z, a.z, fmaf(a.w, a.w, s2))));
          e2 = fmaf(d0, d0, fmaf(d1, d1, fmaf(d2, d2, fmaf(d3, d3, e2))));
          const uint32_t addr = x_base + (uint32_t)(c >> 6) * TX_SLOT_BYTES + (uint32_t)R * 128u +
                                ((((uint32_t)(c & 63) >> 3) ^ ((uint32_t)R & 7u)) << 4) + (uint32_t)(c & 7) * 2u;
          asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(*reinterpret_cast<const uint32_t*>(&h0)),
                       "r"(*reinterpret_cast<const uint32_t*>(&h1)) : "memory");
        }
      }
      s2 = warp_sum(s2); e2 = warp_sum(e2);
      if (lane == 0) ms->rowinfo[R] = (tc_bf16_up(e2) << 16) | tc_bf16_up(s2);
    }
    fence_proxy_async();                 // generic-proxy smem writes -> visible to the tensor core (async proxy)
    tx_wg_sync();

#pragma unroll 1
    for (int l = 0; l < L; ++l) {
      // ---- S = X . C_l^T over the k chunks; a stage is released as soon as the MMAs that read it have completed
      float acc[128];
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

      // ---- score: h = T - S / 2^s in place; columns 8 jb + 2 q4 + {0, 1} of rows r0 (acc[4 jb + 0..1]) and r1 (acc[4 jb + 2..3])
      const TcLevelConst lc = p.hdr->lv[l];
      const float ninv = -1.f / lc.sc;
      if (l == 0) {
#pragma unroll
        for (int jb = 0; jb < 32; ++jb) {
          const float2 t = __ldg(reinterpret_cast<const float2*>(p.hcc + 8 * jb + 2 * q4));
          acc[4 * jb + 0] = fmaf(acc[4 * jb + 0], ninv, t.x); acc[4 * jb + 1] = fmaf(acc[4 * jb + 1], ninv, t.y);
          acc[4 * jb + 2] = fmaf(acc[4 * jb + 2], ninv, t.x); acc[4 * jb + 3] = fmaf(acc[4 * jb + 3], ninv, t.y);
        }
      } else {
        // Gram rows of the previous levels' ids, table (j, l) at gram + (l (l - 1) / 2 + j) 256^2, summed in level order
        const float* g0 = p.gram + (size_t)(l * (l - 1) / 2) * TC_K * TC_K + 2 * q4;
        const float* a0 = g0 + (uint32_t)ids8[r0] * TC_K;
        const float* a1 = g0 + (uint32_t)ids8[r1] * TC_K;
#pragma unroll
        for (int jb = 0; jb < 32; ++jb) {
          float2 t0 = __ldg(reinterpret_cast<const float2*>(a0 + 8 * jb));
          float2 t1 = __ldg(reinterpret_cast<const float2*>(a1 + 8 * jb));
#pragma unroll 1
          for (int j = 1; j < l; ++j) {
            const float* gj = g0 + (size_t)j * TC_K * TC_K + 8 * jb;
            const float2 u0 = __ldg(reinterpret_cast<const float2*>(gj + (uint32_t)ids8[j * TX_R + r0] * TC_K));
            const float2 u1 = __ldg(reinterpret_cast<const float2*>(gj + (uint32_t)ids8[j * TX_R + r1] * TC_K));
            t0.x += u0.x; t0.y += u0.y; t1.x += u1.x; t1.y += u1.y;
          }
          acc[4 * jb + 0] = fmaf(acc[4 * jb + 0], ninv, t0.x); acc[4 * jb + 1] = fmaf(acc[4 * jb + 1], ninv, t0.y);
          acc[4 * jb + 2] = fmaf(acc[4 * jb + 2], ninv, t1.x); acc[4 * jb + 3] = fmaf(acc[4 * jb + 3], ninv, t1.y);
        }
      }
      // ---- row minimum over the quad's 256 codes, then the candidate bits (NaN keeps the code)
      float m0 = INFINITY, m1 = INFINITY;
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
      const float thr0 = m0 + tx_margin(lc, ms->rowinfo[r0]), thr1 = m1 + tx_margin(lc, ms->rowinfo[r1]);
      uint32_t w0[8], w1[8];
      int cnt0 = 0, cnt1 = 0, first0 = 256, first1 = 256;
#pragma unroll
      for (int w = 7; w >= 0; --w) {
        uint32_t b0 = 0u, b1 = 0u;
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
        w0[w] = b0; w1[w] = b1;
        cnt0 += __popc(b0); cnt1 += __popc(b1);
        first0 = b0 ? w * 32 + __ffs(b0) - 1 : first0;
        first1 = b1 ? w * 32 + __ffs(b1) - 1 : first1;
      }
      if (q4 < 2) {                                         // lane 4i + 0 finalises row r0, lane 4i + 1 row r1
        const int r = q4 ? r1 : r0, cnt = q4 ? cnt1 : cnt0, first = q4 ? first1 : first0;
        const int grow = row0 + r;
        if (cnt != 1 && grow < p.B) {
          const uint32_t qi = atomicAdd(&ms->fl_count, 1u);
          ms->flist[qi] = (unsigned char)r;
#pragma unroll
          for (int w = 0; w < 8; ++w) ms->cmask[r][w] = q4 ? w1[w] : w0[w];
        } else {
          const int my_id = first > 255 ? 0 : first;
          ids8[l * TX_R + r] = (unsigned char)my_id;
          if (grow < p.B) p.ids[(int64_t)grow * L + l] = my_id;
        }
      }
      tx_wg_sync();                                         // the re-rank queue of the tile is complete

      // ---- exact re-rank of the queued rows, any warp takes the next one (same arithmetic as rq_simt.cu: sequential fp32
      // residual, (xx + cc) - 2 dot, candidates in ascending index order with a strict '<': first index wins ties).
      // Lane covers elements 128 i + 4 lane .. +3 of a row (6 x LDG.128 per row).
      {
        const float* ccl = p.cc + l * TC_K;
        const float* cl = p.cbf + (size_t)l * TC_K * D;
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
          const uint32_t word = ms->cmask[rrow][lane & 7];     // lane w < 8 holds candidate word w
          // first two candidates (ascending code order): their rows, the x row and the first prior code are ALL requested
          // before anything is consumed -- one or two L2 round trips instead of four dependent ones
          uint32_t wcur = 0, mwd = 0;
          int w = 0;
          auto next_cand = [&]() -> int {                     // -1 when the candidate words are exhausted
            while (mwd == 0u) {
              if (w >= 8) return -1;
              mwd = __shfl_sync(0xffffffffu, word, w);
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
          if (l > 0) ld_row(p.cbf + (size_t)ids8[rrow] * D, vb);          // first prior code travels in vb
          if (ka >= 0) ld_row(cl + (size_t)ka * D, va);
#pragma unroll 1
          for (int j = 0; j < l; ++j) {
#pragma unroll
            for (int i = 0; i < 6; ++i) { res[i].x -= vb[i].x; res[i].y -= vb[i].y; res[i].z -= vb[i].z; res[i].w -= vb[i].w; }   // rqvae.py:130, level order
            if (j + 1 < l) ld_row(p.cbf + ((size_t)(j + 1) * TC_K + (size_t)ids8[(j + 1) * TX_R + rrow]) * D, vb);
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
            const float dist_a = (xx + cca) - 2.f * da;       // quantize.py:113-117
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
          if (besti > 255) besti = firsti < 0 ? 0 : firsti;   // all-NaN distances: keep a valid code
          if (lane == 0) {
            ids8[l * TX_R + rrow] = (unsigned char)besti;
            p.ids[(int64_t)rgrow * L + l] = besti;
          }
          ++n_rows; n_cand += nc; n_many += (nc >= 3);
        }
        if (p.stats && lane == 0 && n_rows) {
          atomicAdd(p.stats + 0, n_rows);
          atomicAdd(p.stats + 1, n_cand);
          atomicAdd(p.stats + 2, n_many);
        }
      }
      tx_wg_sync();                                         // every id of the level is in ids8[]; the queue is drained
      if (tid == 0) { ms->fl_count = 0; ms->fl_next = 0; }
      tx_wg_sync();
    }
  }
}

int tcx_run(const float* x, int64_t ldx, int B, const void* state, int D, int L, int64_t* ids, int* stats, int sm_count,
            cudaStream_t st) {
  const char* base = reinterpret_cast<const char*>(state);
  TxParams p{};
  p.x = x; p.ldx = ldx; p.B = B; p.D = D; p.L = L; p.nkc = D / TC_KC;
  p.ntiles = (B + TX_R - 1) / TX_R;
  p.hdr = reinterpret_cast<const TcHeader*>(base);
  p.cc = reinterpret_cast<const float*>(base + tc_off_cc(TC_K, L));
  p.hcc = reinterpret_cast<const float*>(base + tc_off_hcc(TC_K, L));
  p.gram = reinterpret_cast<const float*>(base + tc_off_gram(TC_K, L));
  p.cbf = reinterpret_cast<const float*>(base + tc_off_cbf(TC_K, L));
  p.blob = reinterpret_cast<const unsigned char*>(base + tc_off_blob(D, TC_K, L));
  p.ids = ids; p.stats = stats;
  // shared memory: x image + codebook ring + fixed part + id bytes of L levels; the ring gets as many 32 KB stages
  // (<= TX_NB_MAX) as fit under the 227 KB limit (2 at D = 768 with 8 levels, 4 with 3 levels)
  const size_t fixed = (size_t)p.nkc * TX_SLOT_BYTES + sizeof(TxSmem) + (size_t)L * TX_R;
  int nbs = TX_NB_MAX;
  while (nbs > 2 && fixed + (size_t)nbs * TX_STAGE_BYTES > TX_SMEM_LIMIT) --nbs;
  p.nb = nbs;
  const size_t smem = fixed + (size_t)nbs * TX_STAGE_BYTES;
  RQB_CUDA(cudaFuncSetAttribute(rq_tcx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = p.ntiles < sm_count ? p.ntiles : sm_count;
  rq_tcx_kernel<<<grid, TX_THREADS, smem, st>>>(p);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}
