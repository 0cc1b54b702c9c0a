// Exact-fp32 fused L-level residual-quantisation kernels (CUDA cores, sm_90a).
//
// One launch runs all L Quantize levels of modules/rqvae.py:125-132 for a tile of rows:
//   * the residual tile lives in shared memory for the whole kernel (never written to HBM unless the
//     caller asks for the `residuals` output),
//   * the (pre-transposed) codebooks are streamed through a 3-stage shared-memory ring by the TMA
//     engine (cp.async.bulk + mbarrier),
//   * every thread owns a TM x TN register tile of the [rows x codes] score matrix, rows map to warps and
//     codes to lanes so the per-row argmin is a warp-shuffle reduction (first index wins ties),
//   * the per-level epilogue (gather of the winning code, STE / rotation-trick output, QuantizeLoss,
//     ||emb||, residual update) is fused behind it.
// This is the always-exact path; rq_tc.cu holds the tensor-core (tcgen05) candidate filter that reuses
// the same exact arithmetic for its re-rank.
#include "common.cuh"
#include <cfloat>
#include <cmath>
#include <cstdlib>

#define RQ_THREADS 256
#define RQ_BK 16
#define RQ_NST 3

enum { RQ_MODE_EVAL = 0, RQ_MODE_STE = 2, RQ_MODE_ROT = 3, RQ_MODE_KMEANS = 4 };

struct RqParams {
  const float* x;
  int64_t ldx;
  const float* cb[RQB_MAX_LEVELS];  // codebooks [K][D] as the caller holds them
  const float* ct;                  // workspace: transposed, zero padded [L][Dp][Kp]
  const float* cc;                  // workspace: ||c||^2, +inf on padded codes [L][Kp]
  int B, D, K, L, Dp, Kp;
  float beta;
  int mode;
  int64_t* ids;     // [B][L]
  float* emb;       // [L][B][D]
  float* resid;     // [L][B][D]
  float* emb_sum;   // [B][D]
  float* emb_norm;  // [B][L]
  float* loss;      // [B]
  double* km_sums;  // [K][D]
  int* km_counts;   // [K]
  int64_t* km_assign;  // [B]
};

// ------------------------------------------------------------------------------------------------ prep
// CT[l][d][k] = C_l[k][d] (zero padded), cc[l][k] = sum_d C_l[k][d]^2 (+inf on padding).
struct PrepParams {
  const float* cb[RQB_MAX_LEVELS];
  float* ct;
  float* cc;
  int D, K, Dp, Kp;
};

__global__ void rq_prep_transpose_kernel(PrepParams p) {
  __shared__ float tile[32][33];
  const int l = blockIdx.z;
  const int k0 = blockIdx.x * 32, d0 = blockIdx.y * 32;
  const float* __restrict__ c = p.cb[l];
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int k = k0 + i, d = d0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < p.K && d < p.D) ? c[(int64_t)k * p.D + d] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int d = d0 + i, k = k0 + threadIdx.x;
    if (d < p.Dp && k < p.Kp) p.ct[((int64_t)l * p.Dp + d) * p.Kp + k] = tile[threadIdx.x][i];
  }
}

__global__ void rq_prep_norm_kernel(PrepParams p) {
  const int l = blockIdx.y;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= p.Kp) return;
  float s = 0.f;
  if (warp < p.K) {
    const float* __restrict__ c = p.cb[l] + (int64_t)warp * p.D;
    for (int d = lane; d < p.D; d += 32) s = fmaf(c[d], c[d], s);
    s = warp_sum(s);
  } else {
    s = INFINITY;
  }
  if (lane == 0) p.cc[(int64_t)l * p.Kp + warp] = s;
}

// ------------------------------------------------------------------------------------------------ forward
template <int TM, int TN, bool DIRECT>
__global__ void __launch_bounds__(RQ_THREADS, 1) rq_fused_kernel(RqParams p) {
  constexpr int BM = 8 * TM;
  constexpr int BN = 32 * TN;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int RS = p.Dp + 4;  // padded row stride of the residual tile (floats, keeps 16B alignment)
  float* Bs = reinterpret_cast<float*>(smem_raw);            // [NST][BK][BN]
  float* R = Bs + RQ_NST * RQ_BK * BN;                       // [BM][RS]
  uint64_t* full = reinterpret_cast<uint64_t*>(R + BM * RS);  // [NST]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row0 = blockIdx.x * BM;

  const int nTiles = p.Kp / BN;
  const int nChunks = p.Dp / RQ_BK;
  const int perLevel = nTiles * nChunks;
  const int total = p.L * perLevel;
  const uint32_t stage_bytes = RQ_BK * BN * sizeof(float);

  auto issue = [&](int g) {  // called by thread 0: TMA bulk copy of chunk g into stage g % NST
    const int st = g % RQ_NST;
    const int l = g / perLevel, rem = g % perLevel;
    const int tile = rem / nChunks, c = rem % nChunks;
    float* dst = Bs + st * (RQ_BK * BN);
    const float* src = p.ct + ((int64_t)l * p.Dp + (int64_t)c * RQ_BK) * p.Kp + tile * BN;
    mbar_expect_tx(&full[st], stage_bytes);
    if (BN == p.Kp) {
      bulk_g2s(dst, src, stage_bytes, &full[st]);
    } else {
#pragma unroll 1
      for (int r = 0; r < RQ_BK; ++r) bulk_g2s(dst + r * BN, src + (int64_t)r * p.Kp, BN * sizeof(float), &full[st]);
    }
  };

  if (tid == 0) {
    for (int s = 0; s < RQ_NST; ++s) mbar_init(&full[s], 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    for (int g = 0; g < RQ_NST && g < total; ++g) issue(g);
  }

  // ---- load the row tile (zero padded) -------------------------------------------------------------
  {
    const int D4 = p.Dp >> 2;
    const bool vec = ((p.ldx & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.x) & 15) == 0) && ((p.D & 3) == 0);
    for (int idx = tid; idx < BM * D4; idx += RQ_THREADS) {
      const int r = idx / D4, d = (idx - r * D4) << 2;
      const int row = row0 + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < p.B) {
        const float* src = p.x + (int64_t)row * p.ldx + d;
        if (vec && d + 3 < p.D) {
          v = __ldg(reinterpret_cast<const float4*>(src));
        } else {
          if (d + 0 < p.D) v.x = __ldg(src + 0);
          if (d + 1 < p.D) v.y = __ldg(src + 1);
          if (d + 2 < p.D) v.z = __ldg(src + 2);
          if (d + 3 < p.D) v.w = __ldg(src + 3);
        }
      }
      *reinterpret_cast<float4*>(R + r * RS + d) = v;
    }
  }
  __syncthreads();

  float* Rw = R + (warp * TM) * RS;  // this warp's TM rows; only this warp ever touches them again
  float xx[TM], loss_acc[TM];
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    float s = 0.f;
    for (int d = lane; d < p.D; d += 32) s = fmaf(Rw[i * RS + d], Rw[i * RS + d], s);
    xx[i] = warp_sum(s);
    loss_acc[i] = 0.f;
  }

  int g = 0;  // running chunk counter (ring position / parity)
  for (int l = 0; l < p.L; ++l) {
    float best_v[TM];
    int best_i[TM];
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      best_v[i] = INFINITY;
      best_i[i] = 0x7fffffff;
    }
    for (int tile = 0; tile < nTiles; ++tile) {
      float acc[TM][TN];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

      for (int c = 0; c < nChunks; ++c, ++g) {
        const int st = g % RQ_NST;
        mbar_wait(&full[st], (g / RQ_NST) & 1);
        const float* Bst = Bs + st * (RQ_BK * BN) + lane * TN;
        const float* Ac = Rw + c * RQ_BK;
#pragma unroll
        for (int dd = 0; dd < RQ_BK; dd += 4) {
          float4 a[TM];
#pragma unroll
          for (int i = 0; i < TM; ++i) a[i] = *reinterpret_cast<const float4*>(Ac + i * RS + dd);
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            float b[TN];
            const float* bp = Bst + (dd + t) * BN;
            if constexpr (TN == 8) {
              float4 b0 = *reinterpret_cast<const float4*>(bp), b1 = *reinterpret_cast<const float4*>(bp + 4);
              b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
              b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
            } else if constexpr (TN == 4) {
              float4 b0 = *reinterpret_cast<const float4*>(bp);
              b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
            } else if constexpr (TN == 2) {
              float2 b0 = *reinterpret_cast<const float2*>(bp);
              b[0] = b0.x; b[1] = b0.y;
            } else {
              b[0] = bp[0];
            }
#pragma unroll
            for (int i = 0; i < TM; ++i) {
              const float av = t == 0 ? a[i].x : (t == 1 ? a[i].y : (t == 2 ? a[i].z : a[i].w));
#pragma unroll
              for (int j = 0; j < TN; ++j) {
                if constexpr (DIRECT) {
                  const float df = av - b[j];
                  acc[i][j] = fmaf(df, df, acc[i][j]);
                } else {
                  acc[i][j] = fmaf(av, b[j], acc[i][j]);
                }
              }
            }
          }
        }
        __syncthreads();  // every warp is done with stage st
        if (tid == 0 && g + RQ_NST < total) issue(g + RQ_NST);
      }
      // ---- tile epilogue: dist = (xx + cc) - 2 dot   (quantize.py:113-117), running first-index argmin
      const int kbase = tile * BN + lane * TN;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int k = kbase + j;
        float ccv = 0.f;
        if constexpr (!DIRECT) ccv = __ldg(p.cc + (int64_t)l * p.Kp + k);
#pragma unroll
        for (int i = 0; i < TM; ++i) {
          float dist;
          if constexpr (DIRECT) {
            dist = (k < p.K) ? acc[i][j] : INFINITY;
          } else {
            dist = (xx[i] + ccv) - 2.f * acc[i][j];
          }
          if (dist < best_v[i]) {
            best_v[i] = dist;
            best_i[i] = k;
          }
        }
      }
    }

    // ---- per-row epilogue (this warp's rows only) ---------------------------------------------------
#pragma unroll 1
    for (int i = 0; i < TM; ++i) {
      float bv = best_v[i];
      int bi = best_i[i];
      warp_argmin(bv, bi);
      if (bi >= p.K) bi = 0;  // all-NaN row: keep memory-safe
      const int row = row0 + warp * TM + i;
      if (row >= p.B) continue;  // warp-uniform
      float* Rrow = Rw + i * RS;

      if (p.mode == RQ_MODE_KMEANS) {
        if (lane == 0) {
          p.km_assign[row] = bi;
          atomicAdd(p.km_counts + bi, 1);
        }
        double* srow = p.km_sums + (int64_t)bi * p.D;
        for (int d = lane; d < p.D; d += 32) atomicAdd(srow + d, (double)Rrow[d]);
        continue;
      }

      const float* __restrict__ e_ptr = p.cb[l] + (int64_t)bi * p.D;
      float* emb_o = p.emb ? p.emb + ((int64_t)l * p.B + row) * p.D : nullptr;
      float* res_o = p.resid ? p.resid + ((int64_t)l * p.B + row) * p.D : nullptr;
      float* sum_o = p.emb_sum ? p.emb_sum + (int64_t)row * p.D : nullptr;

      // rotation trick scalars (quantize.py:140-153, 34-50)
      float rnorm = 0.f, enorm = 0.f, wn = 1.f, rw = 0.f, ru = 0.f, scale = 1.f, ud = 1.f, qd = 1.f;
      if (p.mode == RQ_MODE_ROT) {
        float rr = 0.f, ee = 0.f;
        for (int d = lane; d < p.D; d += 32) {
          const float r = Rrow[d], e = __ldg(e_ptr + d);
          rr = fmaf(r, r, rr);
          ee = fmaf(e, e, ee);
        }
        rnorm = sqrtf(warp_sum(rr));
        enorm = sqrtf(warp_sum(ee));
        ud = rnorm + 1e-8f;
        qd = enorm + 1e-8f;
        float ww = 0.f;
        for (int d = lane; d < p.D; d += 32) {
          const float w = Rrow[d] / ud + __ldg(e_ptr + d) / qd;
          ww = fmaf(w, w, ww);
        }
        wn = fmaxf(sqrtf(warp_sum(ww)), 1e-6f);
        for (int d = lane; d < p.D; d += 32) {
          const float r = Rrow[d];
          const float u = r / ud, q = __ldg(e_ptr + d) / qd;
          const float w = (u + q) / wn;
          rw = fmaf(r, w, rw);
          ru = fmaf(r, u, ru);
        }
        rw = warp_sum(rw);
        ru = warp_sum(ru);
        scale = enorm / (rnorm + 1e-6f);
      }

      float s = 0.f, nn = 0.f, xn = 0.f;
      for (int d = lane; d < p.D; d += 32) {
        const float r = Rrow[d], e = __ldg(e_ptr + d);
        const float df = r - e;
        s = fmaf(df, df, s);
        float eo;
        if (p.mode == RQ_MODE_EVAL) {
          eo = e;                              // quantize.py:160
        } else if (p.mode == RQ_MODE_STE) {
          eo = r + (e - r);                    // quantize.py:139
        } else {
          const float u = r / ud, q = e / qd;
          const float w = (u + q) / wn;
          eo = ((r - 2.f * (rw * w)) + 2.f * (ru * q)) * scale;   // quantize.py:41-50,147-153
        }
        if (res_o) res_o[d] = r;
        if (emb_o) emb_o[d] = eo;
        if (sum_o) sum_o[d] = (l == 0) ? eo : (sum_o[d] + eo);
        const float rn = r - eo;               // rqvae.py:130
        Rrow[d] = rn;
        nn = fmaf(eo, eo, nn);
        xn = fmaf(rn, rn, xn);
      }
      s = warp_sum(s);
      nn = warp_sum(nn);
      xx[i] = warp_sum(xn);
      loss_acc[i] += s + p.beta * s;           // loss.py:39-41 (two identical, separately rounded terms)
      if (lane == 0) {
        if (p.ids) p.ids[(int64_t)row * p.L + l] = bi;
        if (p.emb_norm) p.emb_norm[(int64_t)row * p.L + l] = sqrtf(nn);
      }
    }
    __syncwarp();
  }
  if (p.loss && p.mode != RQ_MODE_KMEANS) {
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int row = row0 + warp * TM + i;
      if (lane == 0 && row < p.B) p.loss[row] = loss_acc[i];
    }
  }
}

// ------------------------------------------------------------------------------------------------ forward from given ids
// The per-row epilogue of rq_fused_kernel on its own: with the ids already known (from the tensor-core tokeniser, whose ids are
// those of the exact kernel) the embeddings / residuals / sums / norms / loss of all L levels are a streaming pass -- one warp
// per row, the residual in shared memory, the SAME loops and reductions as above, hence bit-identical outputs.  This is what
// makes the training-mode forward of a large batch HBM-bound instead of CUDA-core-FLOP-bound (65 536 x 768, L = 3: 5.7 ms fused).
__global__ void rq_replay_kernel(RqParams p) {
  extern __shared__ __align__(16) float rsm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  float* Rrow = rsm + (size_t)warp * p.D;
  for (int row = blockIdx.x * wpb + warp; row < p.B; row += gridDim.x * wpb) {
    const float* xr = p.x + (int64_t)row * p.ldx;
    for (int d = lane; d < p.D; d += 32) Rrow[d] = __ldg(xr + d);
    __syncwarp();
    float loss_acc = 0.f;
    for (int l = 0; l < p.L; ++l) {
      int64_t bi = p.ids[(int64_t)row * p.L + l];
      if (bi < 0 || bi >= p.K) bi = 0;                        // memory-safe on a corrupt id
      const float* __restrict__ e_ptr = p.cb[l] + bi * p.D;
      float* emb_o = p.emb ? p.emb + ((int64_t)l * p.B + row) * p.D : nullptr;
      float* res_o = p.resid ? p.resid + ((int64_t)l * p.B + row) * p.D : nullptr;
      float* sum_o = p.emb_sum ? p.emb_sum + (int64_t)row * p.D : nullptr;
      float rnorm = 0.f, enorm = 0.f, wn = 1.f, rw = 0.f, ru = 0.f, scale = 1.f, ud = 1.f, qd = 1.f;
      if (p.mode == RQ_MODE_ROT) {                            // quantize.py:140-153, 34-50
        float rr = 0.f, ee = 0.f;
        for (int d = lane; d < p.D; d += 32) {
          const float r = Rrow[d], e = __ldg(e_ptr + d);
          rr = fmaf(r, r, rr);
          ee = fmaf(e, e, ee);
        }
        rnorm = sqrtf(warp_sum(rr));
        enorm = sqrtf(warp_sum(ee));
        ud = rnorm + 1e-8f;
        qd = enorm + 1e-8f;
        float ww = 0.f;
        for (int d = lane; d < p.D; d += 32) {
          const float w = Rrow[d] / ud + __ldg(e_ptr + d) / qd;
          ww = fmaf(w, w, ww);
        }
        wn = fmaxf(sqrtf(warp_sum(ww)), 1e-6f);
        for (int d = lane; d < p.D; d += 32) {
          const float r = Rrow[d];
          const float u = r / ud, q = __ldg(e_ptr + d) / qd;
          const float w = (u + q) / wn;
          rw = fmaf(r, w, rw);
          ru = fmaf(r, u, ru);
        }
        rw = warp_sum(rw);
        ru = warp_sum(ru);
        scale = enorm / (rnorm + 1e-6f);
      }
      float s = 0.f, nn = 0.f;
      for (int d = lane; d < p.D; d += 32) {
        const float r = Rrow[d], e = __ldg(e_ptr + d);
        const float df = r - e;
        s = fmaf(df, df, s);
        float eo;
        if (p.mode == RQ_MODE_EVAL) {
          eo = e;
        } else if (p.mode == RQ_MODE_STE) {
          eo = r + (e - r);
        } else {
          const float u = r / ud, q = e / qd;
          const float w = (u + q) / wn;
          eo = ((r - 2.f * (rw * w)) + 2.f * (ru * q)) * scale;
        }
        if (res_o) res_o[d] = r;
        if (emb_o) emb_o[d] = eo;
        if (sum_o) sum_o[d] = (l == 0) ? eo : (sum_o[d] + eo);
        Rrow[d] = r - eo;
        nn = fmaf(eo, eo, nn);
      }
      s = warp_sum(s);
      nn = warp_sum(nn);
      loss_acc += s + p.beta * s;
      if (lane == 0 && p.emb_norm) p.emb_norm[(int64_t)row * p.L + l] = sqrtf(nn);
      __syncwarp();
    }
    if (lane == 0 && p.loss) p.loss[row] = loss_acc;
  }
}

// ------------------------------------------------------------------------------------------------ backward
struct RqBwdParams {
  const float* x;
  int64_t ldx;
  const float* cb[RQB_MAX_LEVELS];
  const int64_t* ids;  // [B][L]
  int B, D, K, L;
  float beta;
  int mode;
  const float* g_emb;  // grad wrt embeddings, element strides (sB, sD, sL); nullable
  int64_t ge_sB, ge_sD, ge_sL;
  const float* g_res;  // grad wrt residuals output; nullable
  int64_t gr_sB, gr_sD, gr_sL;
  const float* g_loss;  // grad wrt quantize_loss [B]; nullable
  int64_t gl_sB;
  float* g_x;          // [B][D]
  float* g_cb[RQB_MAX_LEVELS];  // [K][D], accumulated with atomics (caller zero-initialises)
};

// one warp per row; recomputes the forward residual chain (bit-identical arithmetic to rq_fused_kernel),
// then walks the levels backwards (formulas: SURVEY A.3, checked against reference autograd in tests/golden)
__global__ void rq_bwd_kernel(RqBwdParams p) {
  extern __shared__ __align__(16) float bsm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  float* rs = bsm + (size_t)warp * p.L * p.D;  // residual entering each level [L][D]
  float* gn = bsm + (size_t)wpb * p.L * p.D + (size_t)warp * p.D;  // grad wrt residual of the next level [D]

  for (int row = blockIdx.x * wpb + warp; row < p.B; row += gridDim.x * wpb) {
    const float* xr = p.x + (int64_t)row * p.ldx;
    for (int d = lane; d < p.D; d += 32) rs[d] = __ldg(xr + d);
    __syncwarp();
    // ---- forward recompute ----
    for (int l = 0; l + 1 < p.L; ++l) {
      const float* __restrict__ e_ptr = p.cb[l] + p.ids[(int64_t)row * p.L + l] * p.D;
      const float* r_in = rs + (size_t)l * p.D;
      float* r_out = rs + (size_t)(l + 1) * p.D;
      float wn = 1.f, rw = 0.f, ru = 0.f, scale = 1.f, ud = 1.f, qd = 1.f;
      if (p.mode == RQ_MODE_ROT) {
        float rr = 0.f, ee = 0.f;
        for (int d = lane; d < p.D; d += 32) {
          const float r = r_in[d], e = __ldg(e_ptr + d);
          rr = fmaf(r, r, rr);
          ee = fmaf(e, e, ee);
        }
        const float rnorm = sqrtf(warp_sum(rr)), enorm = sqrtf(warp_sum(ee));
        ud = rnorm + 1e-8f;
        qd = enorm + 1e-8f;
        float ww = 0.f;
        for (int d = lane; d < p.D; d += 32) {
          const float w = r_in[d] / ud + __ldg(e_ptr + d) / qd;
          ww = fmaf(w, w, ww);
        }
        wn = fmaxf(sqrtf(warp_sum(ww)), 1e-6f);
        for (int d = lane; d < p.D; d += 32) {
          const float r = r_in[d];
          const float u = r / ud, q = __ldg(e_ptr + d) / qd;
          rw = fmaf(r, (u + q) / wn, rw);
          ru = fmaf(r, u, ru);
        }
        rw = warp_sum(rw);
        ru = warp_sum(ru);
        scale = enorm / (rnorm + 1e-6f);
      }
      for (int d = lane; d < p.D; d += 32) {
        const float r = r_in[d], e = __ldg(e_ptr + d);
        float eo;
        if (p.mode == RQ_MODE_EVAL) eo = e;
        else if (p.mode == RQ_MODE_STE) eo = r + (e - r);
        else {
          const float u = r / ud, q = e / qd;
          eo = ((r - 2.f * (rw * ((u + q) / wn))) + 2.f * (ru * q)) * scale;
        }
        r_out[d] = r - eo;
      }
      __syncwarp();
    }
    // ---- backward over levels ----
    for (int d = lane; d < p.D; d += 32) gn[d] = 0.f;
    const float gamma = p.g_loss ? __ldg(p.g_loss + (int64_t)row * p.gl_sB) : 0.f;
    for (int l = p.L - 1; l >= 0; --l) {
      const int64_t id = p.ids[(int64_t)row * p.L + l];
      const float* __restrict__ e_ptr = p.cb[l] + id * p.D;
      float* gc = p.g_cb[l] ? p.g_cb[l] + id * p.D : nullptr;
      const float* r_in = rs + (size_t)l * p.D;
      const float* ge = p.g_emb ? p.g_emb + (int64_t)row * p.ge_sB + (int64_t)l * p.ge_sL : nullptr;
      const float* gr = p.g_res ? p.g_res + (int64_t)row * p.gr_sB + (int64_t)l * p.gr_sL : nullptr;
      float lam = 1.f, wn = 1.f, ud = 1.f, qd = 1.f, gw = 0.f, gq = 0.f;
      if (p.mode == RQ_MODE_ROT) {
        float rr = 0.f, ee = 0.f;
        for (int d = lane; d < p.D; d += 32) {
          const float r = r_in[d], e = __ldg(e_ptr + d);
          rr = fmaf(r, r, rr);
          ee = fmaf(e, e, ee);
        }
        const float rnorm = sqrtf(warp_sum(rr)), enorm = sqrtf(warp_sum(ee));
        ud = rnorm + 1e-8f;
        qd = enorm + 1e-8f;
        lam = enorm / (rnorm + 1e-6f);
        float ww = 0.f;
        for (int d = lane; d < p.D; d += 32) {
          const float w = r_in[d] / ud + __ldg(e_ptr + d) / qd;
          ww = fmaf(w, w, ww);
        }
        wn = fmaxf(sqrtf(warp_sum(ww)), 1e-6f);
        for (int d = lane; d < p.D; d += 32) {
          const float r = r_in[d], e = __ldg(e_ptr + d);
          const float u = r / ud, q = e / qd;
          const float go = ((ge ? __ldg(ge + (int64_t)d * p.ge_sD) : 0.f) - gn[d]) * lam;
          gw = fmaf(go, (u + q) / wn, gw);
          gq = fmaf(go, q, gq);
        }
        gw = warp_sum(gw);
        gq = warp_sum(gq);
      }
      for (int d = lane; d < p.D; d += 32) {
        const float r = r_in[d], e = __ldg(e_ptr + d);
        const float go = (ge ? __ldg(ge + (int64_t)d * p.ge_sD) : 0.f) - gn[d];  // grad wrt emb_out of this level
        float gx = gn[d] + 2.f * p.beta * gamma * (r - e);
        float gcv = 2.f * gamma * (e - r);
        if (p.mode == RQ_MODE_STE) {
          gx += go;
        } else if (p.mode == RQ_MODE_ROT) {
          const float u = r / ud, q = e / qd;
          const float gh = go * lam;
          gx += gh - 2.f * gw * ((u + q) / wn) + 2.f * gq * u;
        } else {
          gcv += go;  // eval-mode lookup: emb_out = codebook[ids]
        }
        if (gr) gx += __ldg(gr + (int64_t)d * p.gr_sD);
        if (gc) atomicAdd(gc + d, gcv);
        gn[d] = gx;
      }
      __syncwarp();
    }
    float* gxo = p.g_x + (int64_t)row * p.D;
    for (int d = lane; d < p.D; d += 32) gxo[d] = gn[d];
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------ k-means finalize
// centroid = mean of assigned rows (fp64 sums -> one rounding), or the reseed row for an empty cluster
// (init/kmeans.py:48-58); shift = max_k ||c_new - c_old||_2 (kmeans.py:68) via atomicMax on the float bits.
__global__ void kmeans_finalize_kernel(const double* sums, const int* counts, const float* x, int64_t ldx,
                                       const int64_t* reseed_rows, float* centroids, int K, int D,
                                       unsigned int* max_shift_bits) {
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= K) return;
  const int cnt = counts[k];
  float sh = 0.f;
  for (int d = lane; d < D; d += 32) {
    float nv;
    if (cnt > 0) {
      nv = (float)(sums[(int64_t)k * D + d] / (double)cnt);
    } else {
      const int64_t rr = reseed_rows ? reseed_rows[k] : -1;
      nv = rr >= 0 ? x[rr * ldx + d] : centroids[(int64_t)k * D + d];
    }
    const float df = nv - centroids[(int64_t)k * D + d];
    sh = fmaf(df, df, sh);
    centroids[(int64_t)k * D + d] = nv;
  }
  sh = sqrtf(warp_sum(sh));
  if (lane == 0) atomicMax(max_shift_bits, __float_as_uint(sh));
}

// ================================================================================================ host side
static int pick_tn(int K, int* Kp) {
  int tn;
  if (K <= 32) { tn = 1; *Kp = 32; }
  else if (K <= 64) { tn = 2; *Kp = 64; }
  else if (K <= 128) { tn = 4; *Kp = 128; }
  else { tn = 8; *Kp = (int)rqb_round_up(K, 256); }
  return tn;
}

static size_t fused_smem_bytes(int tm, int tn, int Dp) {
  return (size_t)(RQ_NST * RQ_BK * 32 * tn + 8 * tm * (Dp + 4)) * sizeof(float) + RQ_NST * sizeof(uint64_t) + 64;
}

static int pick_tm(int B, int tn, int Dp) {
  if (const char* e = getenv("RQB200_TM")) {     // tuning knob: force the row-tile height (8, 4, 2 or 1)
    const int f = atoi(e);
    if ((f == 8 || f == 4 || f == 2 || f == 1) && fused_smem_bytes(f, tn, Dp) <= 200 * 1024) return f;
  }
  // With a short K loop (D <= 64: at most 4 chunks per level) the 8x8 register tile costs occupancy (168 regs -> one CTA
  // per SM) without paying back in FMA efficiency, so TM = 4 is used there.
  int tm = (Dp <= 64) ? 4 : 8;
  while (tm >= 1 && fused_smem_bytes(tm, tn, Dp) > 200 * 1024) tm >>= 1;
  if (tm < 1) return 0;
  while (tm > 1 && (B + 8 * tm - 1) / (8 * tm) < 132) tm >>= 1;
  return tm;
}

extern "C" size_t rqb200_rq_workspace_bytes(int D, int K, int L) {
  int Kp;
  pick_tn(K, &Kp);
  const int64_t Dp = rqb_round_up(D, RQ_BK);
  return (size_t)L * Dp * Kp * sizeof(float) + (size_t)L * Kp * sizeof(float) + 256;
}

static int run_prep(const float* const* cbs, int D, int K, int L, void* ws, size_t ws_bytes, cudaStream_t st,
                    const float** ct, const float** cc, int* Dp_out, int* Kp_out) {
  int Kp;
  pick_tn(K, &Kp);
  const int Dp = (int)rqb_round_up(D, RQ_BK);
  if (ws_bytes < rqb200_rq_workspace_bytes(D, K, L)) {
    rqb_set_error("workspace too small: %zu < %zu", ws_bytes, rqb200_rq_workspace_bytes(D, K, L));
    return RQB_ERR_WORKSPACE;
  }
  PrepParams pp;
  for (int l = 0; l < L; ++l) pp.cb[l] = cbs[l];
  pp.ct = reinterpret_cast<float*>(ws);
  pp.cc = pp.ct + (size_t)L * Dp * Kp;
  pp.D = D; pp.K = K; pp.Dp = Dp; pp.Kp = Kp;
  dim3 g1(Kp / 32, (Dp + 31) / 32, L), b1(32, 8);
  rq_prep_transpose_kernel<<<g1, b1, 0, st>>>(pp);
  RQB_LAUNCH_CHECK();
  dim3 g2((Kp * 32 + 255) / 256, L);
  rq_prep_norm_kernel<<<g2, 256, 0, st>>>(pp);
  RQB_LAUNCH_CHECK();
  *ct = pp.ct; *cc = pp.cc; *Dp_out = Dp; *Kp_out = Kp;
  return RQB_OK;
}

template <int TM, int TN>
static int launch_fused(const RqParams& p, bool direct, cudaStream_t st) {
  const size_t smem = fused_smem_bytes(TM, TN, p.Dp);
  const int grid = (p.B + 8 * TM - 1) / (8 * TM);
  if (direct) {
    RQB_CUDA(cudaFuncSetAttribute(rq_fused_kernel<TM, TN, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rq_fused_kernel<TM, TN, true><<<grid, RQ_THREADS, smem, st>>>(p);
  } else {
    RQB_CUDA(cudaFuncSetAttribute(rq_fused_kernel<TM, TN, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rq_fused_kernel<TM, TN, false><<<grid, RQ_THREADS, smem, st>>>(p);
  }
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

template <int TN>
static int dispatch_tm(int tm, const RqParams& p, bool direct, cudaStream_t st) {
  switch (tm) {
    case 8: return launch_fused<8, TN>(p, direct, st);
    case 4: return launch_fused<4, TN>(p, direct, st);
    case 2: return launch_fused<2, TN>(p, direct, st);
    default: return launch_fused<1, TN>(p, direct, st);
  }
}

static int dispatch_fused(RqParams& p, bool direct, cudaStream_t st) {
  if (p.B == 0) return RQB_OK;
  int Kp;
  const int tn = pick_tn(p.K, &Kp);
  const int tm = pick_tm(p.B, tn, p.Dp);
  if (tm == 0) {
    rqb_set_error("embed_dim %d too large for the shared-memory residual tile", p.D);
    return RQB_ERR_UNSUPPORTED;
  }
  switch (tn) {
    case 8: return dispatch_tm<8>(tm, p, direct, st);
    case 4: return dispatch_tm<4>(tm, p, direct, st);
    case 2: return dispatch_tm<2>(tm, p, direct, st);
    default: return dispatch_tm<1>(tm, p, direct, st);
  }
}

extern "C" int rqb200_rq_forward(int mode, const float* x, int64_t ldx, const float* const* codebooks, int B, int D,
                                 int K, int L, float beta, int64_t* ids, float* embeddings, float* residuals,
                                 float* emb_sum, float* emb_norms, float* loss, void* workspace, size_t ws_bytes,
                                 void* stream) {
  RQB_CHECK_ARG(mode == RQ_MODE_EVAL || mode == RQ_MODE_STE || mode == RQ_MODE_ROT, "rq_forward: bad mode %d", mode);
  RQB_CHECK_ARG(B >= 0 && D > 0 && K > 0 && L > 0 && L <= RQB_MAX_LEVELS, "rq_forward: bad shape B=%d D=%d K=%d L=%d", B, D, K, L);
  RQB_CHECK_ARG(B == 0 || (x && codebooks && workspace), "rq_forward: null pointer");
  RQB_CHECK_ARG(ldx >= D, "rq_forward: ldx %lld < D %d", (long long)ldx, D);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (B == 0) return RQB_OK;
  RqParams p{};
  int rc = run_prep(codebooks, D, K, L, workspace, ws_bytes, st, &p.ct, &p.cc, &p.Dp, &p.Kp);
  if (rc) return rc;
  p.x = x; p.ldx = ldx;
  for (int l = 0; l < L; ++l) { RQB_CHECK_ARG(codebooks[l], "rq_forward: null codebook %d", l); p.cb[l] = codebooks[l]; }
  p.B = B; p.D = D; p.K = K; p.L = L; p.beta = beta; p.mode = mode;
  p.ids = ids; p.emb = embeddings; p.resid = residuals; p.emb_sum = emb_sum; p.emb_norm = emb_norms; p.loss = loss;
  return dispatch_fused(p, false, st);
}

extern "C" int rqb200_rq_forward_from_ids(int mode, const float* x, int64_t ldx, const float* const* codebooks,
                                          const int64_t* ids, int B, int D, int K, int L, float beta, float* embeddings,
                                          float* residuals, float* emb_sum, float* emb_norms, float* loss, void* stream) {
  RQB_CHECK_ARG(mode == RQ_MODE_EVAL || mode == RQ_MODE_STE || mode == RQ_MODE_ROT, "rq_forward_from_ids: bad mode %d", mode);
  RQB_CHECK_ARG(B >= 0 && D > 0 && K > 0 && L > 0 && L <= RQB_MAX_LEVELS && ldx >= D, "rq_forward_from_ids: bad shape");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(x && codebooks && ids, "rq_forward_from_ids: null pointer");
  RqParams p{};
  p.x = x; p.ldx = ldx;
  for (int l = 0; l < L; ++l) { RQB_CHECK_ARG(codebooks[l], "rq_forward_from_ids: null codebook %d", l); p.cb[l] = codebooks[l]; }
  p.B = B; p.D = D; p.K = K; p.L = L; p.beta = beta; p.mode = mode;
  p.ids = const_cast<int64_t*>(ids);
  p.emb = embeddings; p.resid = residuals; p.emb_sum = emb_sum; p.emb_norm = emb_norms; p.loss = loss;
  int wpb = 8;
  while (wpb > 1 && (size_t)wpb * D * sizeof(float) > 96 * 1024) wpb >>= 1;
  const size_t smem = (size_t)wpb * D * sizeof(float);
  if (smem > 200 * 1024) { rqb_set_error("rq_forward_from_ids: D too large (%d)", D); return RQB_ERR_UNSUPPORTED; }
  RQB_CUDA(cudaFuncSetAttribute(rq_replay_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = (B + wpb - 1) / wpb;
  if (grid > 132 * 8) grid = 132 * 8;
  rq_replay_kernel<<<grid, wpb * 32, smem, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

extern "C" int rqb200_rq_backward(int mode, const float* x, int64_t ldx, const float* const* codebooks,
                                  const int64_t* ids, int B, int D, int K, int L, float beta, const float* g_emb,
                                  int64_t ge_sB, int64_t ge_sD, int64_t ge_sL, const float* g_res, int64_t gr_sB,
                                  int64_t gr_sD, int64_t gr_sL, const float* g_loss, int64_t gl_sB, float* g_x,
                                  float* const* g_codebooks, void* stream) {
  RQB_CHECK_ARG(mode == RQ_MODE_EVAL || mode == RQ_MODE_STE || mode == RQ_MODE_ROT, "rq_backward: bad mode %d", mode);
  RQB_CHECK_ARG(B >= 0 && D > 0 && K > 0 && L > 0 && L <= RQB_MAX_LEVELS, "rq_backward: bad shape");
  if (B == 0) return RQB_OK;
  RQB_CHECK_ARG(x && codebooks && ids && g_x, "rq_backward: null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RqBwdParams p{};
  p.x = x; p.ldx = ldx; p.ids = ids; p.B = B; p.D = D; p.K = K; p.L = L; p.beta = beta; p.mode = mode;
  for (int l = 0; l < L; ++l) { p.cb[l] = codebooks[l]; p.g_cb[l] = g_codebooks ? g_codebooks[l] : nullptr; }
  p.g_emb = g_emb; p.ge_sB = ge_sB; p.ge_sD = ge_sD; p.ge_sL = ge_sL;
  p.g_res = g_res; p.gr_sB = gr_sB; p.gr_sD = gr_sD; p.gr_sL = gr_sL;
  p.g_loss = g_loss; p.gl_sB = gl_sB; p.g_x = g_x;
  int wpb = 8;
  while (wpb > 1 && (size_t)wpb * (L + 1) * D * sizeof(float) > 160 * 1024) wpb >>= 1;
  const size_t smem = (size_t)wpb * (L + 1) * D * sizeof(float);
  if (smem > 200 * 1024) { rqb_set_error("rq_backward: L*D too large (%d x %d)", L, D); return RQB_ERR_UNSUPPORTED; }
  RQB_CUDA(cudaFuncSetAttribute(rq_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = (B + wpb - 1) / wpb;
  if (grid > 132 * 8) grid = 132 * 8;
  rq_bwd_kernel<<<grid, wpb * 32, smem, st>>>(p);
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}

// k-means: one Lloyd assignment pass (init/kmeans.py:39-46) + per-cluster fp64 sums / counts (kmeans.py:48-58).
extern "C" int rqb200_kmeans_assign_accumulate(const float* x, int64_t ldx, const float* centroids, int B, int D, int K,
                                               int64_t* assignment, double* sums, int* counts, void* workspace,
                                               size_t ws_bytes, void* stream) {
  RQB_CHECK_ARG(B >= 0 && D > 0 && K > 0, "kmeans: bad shape");
  RQB_CHECK_ARG(centroids && sums && counts, "kmeans: null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RQB_CUDA(cudaMemsetAsync(sums, 0, (size_t)K * D * sizeof(double), st));
  RQB_CUDA(cudaMemsetAsync(counts, 0, (size_t)K * sizeof(int), st));
  if (B == 0) return RQB_OK;  // an empty shard (x and assignment may be null): zero sums and counts
  RQB_CHECK_ARG(x && assignment && workspace, "kmeans: null pointer");
  RqParams p{};
  const float* cbs[1] = {centroids};
  int rc = run_prep(cbs, D, K, 1, workspace, ws_bytes, st, &p.ct, &p.cc, &p.Dp, &p.Kp);
  if (rc) return rc;
  p.x = x; p.ldx = ldx; p.cb[0] = centroids; p.B = B; p.D = D; p.K = K; p.L = 1; p.mode = RQ_MODE_KMEANS;
  p.km_sums = sums; p.km_counts = counts; p.km_assign = assignment;
  return dispatch_fused(p, true, st);
}

extern "C" int rqb200_kmeans_finalize(const double* sums, const int* counts, const float* x, int64_t ldx,
                                      const int64_t* reseed_rows, float* centroids, int K, int D, float* max_shift,
                                      void* stream) {
  RQB_CHECK_ARG(sums && counts && centroids && max_shift && K > 0 && D > 0, "kmeans_finalize: bad argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RQB_CUDA(cudaMemsetAsync(max_shift, 0, sizeof(float), st));
  kmeans_finalize_kernel<<<(K + 7) / 8, 256, 0, st>>>(sums, counts, x, ldx, reseed_rows, centroids, K, D,
                                                      reinterpret_cast<unsigned int*>(max_shift));
  RQB_LAUNCH_CHECK();
  return RQB_OK;
}
