/* librqb200 -- C ABI of the H100-native RQ-VAE residual-quantisation hot path.
 *
 * The reference (EdoardoBotta/RQ-VAE-Recommender) has no FFI layer: its boundary is the Python module API
 * (modules/quantize.py, modules/rqvae.py, init/kmeans.py, distributions/gumbel.py, modules/encoder.py).
 * This header is the C boundary those replacement modules bind (via ctypes, see
 * rq_vae_recommender_b200/_lib.py and INTEGRATION.md).  Each entry point cites the reference code it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name says host (`const float* const* codebooks` is a HOST
 *     array of L device pointers); row-major storage; strides/leading dimensions are in ELEMENTS;
 *   - no allocation, no ownership transfer: the caller (PyTorch) allocates outputs and workspaces
 *     (sizes from the *_workspace_bytes queries) and keeps them alive until the stream work completes;
 *   - `stream` is a cudaStream_t; all work is enqueued on it, nothing synchronises the host;
 *   - every function returns 0 on success or an RQB_ERR_* code; rqb200_last_error() gives the text
 *     (thread-local).  No exceptions cross the boundary.  No global mutable state besides that string.
 */
#ifndef RQB200_H
#define RQB200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RQB_OK 0
#define RQB_ERR_INVALID 1
#define RQB_ERR_CUDA 2
#define RQB_ERR_UNSUPPORTED 3
#define RQB_ERR_WORKSPACE 4

#define RQB_MAX_LEVELS 8

/* forward modes: numbering of modules/quantize.py:16-20 (QuantizeForwardMode), 0 = eval-mode lookup */
#define RQB_MODE_EVAL 0
#define RQB_MODE_GUMBEL 1
#define RQB_MODE_STE 2
#define RQB_MODE_ROTATION 3

int rqb200_version(void);
const char* rqb200_last_error(void);
int rqb200_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---- fused L-level residual quantisation, exact fp32 -------------------------------------------------
 * Replaces L x Quantize.forward (modules/quantize.py:104-163: distance :113-117, argmin :128, eval lookup
 * :159-161, STE :137-139, rotation trick :140-153 + :34-50, QuantizeLoss modules/loss.py:38-41) chained by
 * RqVae.get_semantic_ids (modules/rqvae.py:122-139: residual update :130, loss accumulation :128).
 * x is the encoder output [B,D] (ldx >= D).  All outputs are optional (NULL = not produced):
 *   ids [B,L] int64; embeddings / residuals [L,B,D] (the Python side returns [B,D,L] views);
 *   emb_sum [B,D] = sum_l emb_out (rqvae.py:146); emb_norms [B,L] = ||emb_out|| (rqvae.py:158); loss [B].
 * Tokenisation (modules/tokenizer/semids.py:125) is mode = EVAL with only `ids`. */
size_t rqb200_rq_workspace_bytes(int D, int K, int L);
int rqb200_rq_forward(int mode, const float* x, int64_t ldx, const float* const* codebooks, int B, int D, int K,
                      int L, float beta, int64_t* ids, float* embeddings, float* residuals, float* emb_sum,
                      float* emb_norms, float* loss, void* workspace, size_t workspace_bytes, void* stream);

/* The same outputs from GIVEN ids (no distance computation): the streaming half of the chain.  With the ids of the
 * tensor-core tokeniser (identical to the exact kernel's) this is how a large training-mode batch runs: tokenise + this pass
 * instead of CUDA-core distances; outputs are bit-identical to rqb200_rq_forward's for the same ids. */
int rqb200_rq_forward_from_ids(int mode, const float* x, int64_t ldx, const float* const* codebooks, const int64_t* ids,
                               int B, int D, int K, int L, float beta, float* embeddings, float* residuals, float* emb_sum,
                               float* emb_norms, float* loss, void* stream);

/* Backward of the above (autograd of quantize.py:130-161 + loss.py:38-41 through the chain rqvae.py:125-132;
 * formulas SURVEY appendix A.3).  Upstream grads come with element strides so expanded / permuted torch
 * tensors need no copy: g_emb[b,d,l] = g_emb[b*ge_sB + d*ge_sD + l*ge_sL] (NULL = zero), same for g_res;
 * g_loss[b*gl_sB].  g_x [B,D] is written; g_codebooks[l] [K,D] are ACCUMULATED (caller zero-fills). */
int rqb200_rq_backward(int mode, const float* x, int64_t ldx, const float* const* codebooks, const int64_t* ids,
                       int B, int D, int K, int L, float beta, const float* g_emb, int64_t ge_sB, int64_t ge_sD,
                       int64_t ge_sL, const float* g_res, int64_t gr_sB, int64_t gr_sD, int64_t gr_sL,
                       const float* g_loss, int64_t gl_sB, float* g_x, float* const* g_codebooks, void* stream);

/* ---- tensor-core tokeniser (wgmma candidate filter + exact fp32 re-rank), see csrc/rq_tc.cu --------
 * Same result contract as rqb200_rq_forward(mode=EVAL, ids only).  `prepare` converts the codebooks once
 * (fp16 copies, norms, inter-level Gram tables) into `state`; `run` consumes x [B,D] fp32.
 * Supported: K = 256 m with 1 <= m <= 8 (256 ... 2048 codes), D a multiple of 64 in 64..768, 1 <= L <= 8.
 * state_bytes grows as K^2 L(L-1)/2 (the Gram tables): ~80 MB at K = 2048, L = 3, D = 768; ~0.55 GB at L = 8. */
size_t rqb200_tokenize_tc_state_bytes(int D, int K, int L);
int rqb200_tokenize_tc_supported(int D, int K, int L);
/* Host only: 32 KB codebook ring stages `run` gives a CTA at this shape (3 or 4, whatever fits in 227 KB of shared memory
 * next to the x image and the candidate words), 0 for an unsupported shape. */
int rqb200_tokenize_tc_ring_stages(int D, int K, int L);
int rqb200_tokenize_tc_prepare(const float* const* codebooks, int D, int K, int L, void* state, size_t state_bytes,
                               void* stream);
int rqb200_tokenize_tc_run(const float* x, int64_t ldx, int B, const void* state, int D, int K, int L,
                           int64_t* ids, int* stats, void* stream);

/* ---- k-means codebook initialisation (init/kmeans.py) ------------------------------------------------
 * assign_accumulate = one Lloyd assignment pass with the direct (x-c)^2 distance of kmeans.py:40-43 plus the
 * per-cluster sums (fp64) and counts that kmeans.py:48-58 derives with a Python loop; in the sharded setting
 * the caller all-reduces sums/counts between the two calls; an empty shard (B = 0, x and assignment may be
 * NULL) contributes zero sums and counts.  finalize writes the new centroids in place
 * (mean, or x[reseed_rows[k]] for an empty cluster, kmeans.py:50-54; reseed_rows may be NULL) and the
 * max centroid shift of kmeans.py:68 into *max_shift (device float). */
int rqb200_kmeans_assign_accumulate(const float* x, int64_t ldx, const float* centroids, int B, int D, int K,
                                    int64_t* assignment, double* sums, int* counts, void* workspace,
                                    size_t workspace_bytes, void* stream);
int rqb200_kmeans_finalize(const double* sums, const int* counts, const float* x, int64_t ldx,
                           const int64_t* reseed_rows, float* centroids, int K, int D, float* max_shift,
                           void* stream);

/* ---- dense fp32 helpers -------------------------------------------------------------------------------
 * sgemm: C = epi(alpha * op(A) op(B) + beta * C), row-major, op = transpose flag; relu and the (mask > 0)
 * epilogue fuse the ReLU forward / backward of modules/encoder.py:27-29.  Also the W@C and gradient GEMMs of
 * the Gumbel path (quantize.py:135). */
int rqb200_sgemm(int transA, int transB, int M, int N, int K, float alpha, const float* A, int64_t lda,
                 const float* B, int64_t ldb, float beta, float* C, int64_t ldc, int relu, const float* mask,
                 int64_t ldmask, void* stream);
int rqb200_row_sqnorm(const float* c, int K, int D, float* out, void* stream);
/* dots [B,K] (= x @ C^T) -> dist in place (quantize.py:113-117) + first-index argmin (quantize.py:128) */
int rqb200_dist_finish(float* dots, const float* x, int64_t ldx, const float* cc, int B, int D, int K, int64_t* ids,
                       void* stream);
/* W = softmax((-dist + G(U)) / T)  (distributions/gumbel.py:8-20 with U injected; quantize.py:132-134) */
int rqb200_gumbel_softmax_fwd(const float* dist, const float* uniform, float* weights, int B, int K,
                              float temperature, void* stream);
int rqb200_gumbel_row_finish(const float* x, int64_t ldx, const float* E, int B, int D, float beta, float* loss,
                             void* stream);
int rqb200_gumbel_bwd_ge(const float* g_out, int64_t go_sB, int64_t go_sD, const float* g_loss, int64_t gl_sB,
                         const float* x, int64_t ldx, const float* E, float* gE, int B, int D, void* stream);
int rqb200_gumbel_bwd_softmax(const float* weights, float* gw_inout, int B, int K, float temperature, float* rowsum,
                              float* colsum, void* stream);
int rqb200_gumbel_bwd_gx(float* acc_inout, const float* x, int64_t ldx, const float* E, const float* g_loss,
                         int64_t gl_sB, const float* rowsum, float beta, int B, int D, void* stream);
int rqb200_gumbel_bwd_gc(float* gC_inout, const float* C, const float* colsum, int K, int D, void* stream);
/* modules/normalize.py:6-7 (F.normalize p=2) and its backward */
int rqb200_l2norm_fwd(const float* x, float* y, float* norms, int B, int D, float eps, void* stream);
int rqb200_l2norm_bwd(const float* gy, const float* y, const float* norms, float* gx, int B, int D, float eps,
                      void* stream);

/* ---- bf16 tensor-core GEMM for the MLPs (modules/encoder.py:23-38), reduced-precision / AMP-like, forward only ---
 * The reference runs these Linears in bf16 when mixed precision is on (train_rqvae.py:36,69).  Operands live in HBM
 * as "images": [tile of 128 rows][64-wide k chunk][128 x 128 B], the exact K-major SWIZZLE_128B shared-memory layout
 * tcgen05 reads, so a pipeline stage is one contiguous TMA bulk copy.  K must be a multiple of 64.
 *   f32_to_bf16_image : fp32 row-major [rows,K] -> image (used for the input x AND for a weight W[N,K]);
 *   gemm_bf16         : Y = act(X W^T), fp32 accumulate; Y is written as the next layer's A image (N % 64 == 0)
 *                       and/or as fp32 row-major [M,N]. */
size_t rqb200_bf16_image_bytes(int rows, int K);
int rqb200_f32_to_bf16_image(const float* x, int64_t ldx, int rows, int K, void* image, void* stream);
int rqb200_gemm_bf16(const void* a_image, const void* w_image, int M, int N, int K, int relu, void* out_image,
                     float* out_f32, int64_t ldo, void* stream);

/* ---- split-precision tensor-core GEMM: fp32-accurate products on the fp16 tensor cores -----------------------------
 * The MLP Linears of modules/encoder.py:23-38 in their default (index-exact) precision and the two GEMMs of a
 * Gumbel-softmax level (modules/quantize.py:113-117,135).  Each operand row is scaled by a power of two and stored as
 * two fp16 images hi + lo (22 significant bits); C = act(A B^T) costs three tcgen05.mma per k-step (hi.hi + lo.hi +
 * hi.lo, fp32 accumulate) and is written as fp32 rows.
 *   split_image_bytes  : bytes of one operand buffer [hi image][lo image][row scales] for a [rows, K] matrix
 *   f32_to_split_image : fp32 [rows, K] (ld = ldx) -> buffer, any K; transposed != 0 reads the operand as x[K, rows]
 *                        (K <= 65535 * 64)
 *   gemm_split         : out[M, N] (ld = ldo) = act(A[M, K] . B[N, K]^T) from two such buffers; an optional mask[M, N]
 *                        zeroes the entries whose mask value is not > 0 (the ReLU' of a backward GEMM) */
size_t rqb200_split_image_bytes(int rows, int K);
int rqb200_f32_to_split_image(const float* x, int64_t ldx, int rows, int K, int transposed, void* image, void* stream);
int rqb200_gemm_split(const void* a_image, const void* b_image, int M, int N, int K, int relu, const float* mask,
                      int64_t ldm, float* out, int64_t ldo, void* stream);
/* split-K schedule for few output tiles and a long contraction (weight gradients, modules/encoder.py backward: M = out,
 * N = in, K = batch): gemm_split_k_slices returns the slice count that fills the SMs; workspace = slices * M * N floats
 * (unused when slices == 1); the partial sums are reduced in a fixed order. */
int rqb200_gemm_split_k_slices(int M, int N, int K);
int rqb200_gemm_split_k(const void* a_image, const void* b_image, int M, int N, int K, int slices, float* workspace,
                        float* out, int64_t ldo, void* stream);

/* ---- corpus id statistics (train_rqvae.py:279-289, modules/tokenizer/semids.py:94-108) ---------------- */
int rqb200_sid_histogram(const int64_t* ids, int B, int L, int K, int64_t* hist /* [L,K], zeroed here */,
                         void* stream);

/* Dedup column of the corpus table, modules/tokenizer/semids.py:94-108: rank[i] = number of rows j < i with the same id tuple
 * (the reference's O(N^2) compare), and in the same pass the diversity statistics of train_rqvae.py:276-283:
 * stats[0] = max rank (max_id_duplicates * N), stats[1] = number of distinct tuples, *entropy = -sum p log p over the distinct
 * tuples.  Direct-table algorithm: needs K^L <= 2^26 (workspace_bytes returns 0 otherwise and the call RQB_ERR_UNSUPPORTED:
 * the caller falls back to a sort).  ids [N,L] int64 row-major; ids outside [0,K) make a row its own group. */
size_t rqb200_sid_dedup_workspace_bytes(int N, int L, int K);
int rqb200_sid_dedup_rank(const int64_t* ids, int N, int L, int K, int64_t* rank /* [N] */, int* stats /* [2] */,
                          double* entropy /* [1] */, void* workspace, size_t workspace_bytes, void* stream);

/* Sequence tokenisation from the corpus table, semids.py:112-146 (`cached_ids[ids]`, -1 under the padding mask,
 * token_type_ids): out[b, s*C + c] = seq_mask[b,s] ? cached_ids[item_ids[b,s], c] : -1; token_type[b, s*C + c] = c.
 * seq_mask (bytes, 0 = padding) and token_type may be null; strides in elements. */
int rqb200_sid_gather(const int64_t* cached_ids, int64_t n_corpus, int C, const int64_t* item_ids, int64_t item_stride,
                      const unsigned char* seq_mask, int64_t mask_stride, int B, int S, int64_t* out /* [B, S*C] */,
                      int64_t* token_type /* [B, S*C] or null */, void* stream);

/* ---- constrained beam search, data side (modules/model.py:169-182 `_check_valid_prefix`, :340-376 the selection step) ----
 * A trie of the corpus id table [N, C] holds its valid prefixes: the prefixes of every row up to its first id outside [0, K)
 * (a prefix holding such an id is never valid; duplicated rows and N = 0 are legal).  Level l holds the distinct l-prefixes in
 * lexicographic order, each node with its last code and the range of its children.  Limits: N < 2^31 - 1, C <= 8, K <= 65536.
 * sid_trie_workspace_bytes : bytes of the trie the search calls read, (4 (C - 1) + 2 C) N plus alignment; arithmetic only, no
 *                            device.  0 outside the limits.
 * sid_trie_scratch_bytes   : bytes of the build's scratch (the row sort and the per-level scans); queries CUB on the current
 *                            device.  0 outside the limits or when the device cannot be queried.
 * sid_trie_build           : corpus id table [N, C] -> the trie in `workspace`.  Sorts on the stream (CUB radix sort and scans)
 *                            and does not synchronise the host; `scratch` may be reused once the stream has passed the build.
 * sid_trie_check           : valid[p] = some corpus row starts with prefix[p, :l]   (one binary search among a node's children per
 *                            level instead of the reference's O(P N l) compare)
 * sid_trie_beam_select     : one launch per hierarchy level h: score kp x nc candidate extensions per batch row (sampled token
 *                            log-probability + parent beam log-probability, -inf when the extended prefix is not in the corpus),
 *                            keep the k best in descending order, gather their ids into out_generated [B, k, h + 1] and return
 *                            the parent beam's global index b * kp + beam (the key/value-cache reorder index).
 *                            Limits: kp * nc <= 1024, k <= 32, h < C <= 8. */
size_t rqb200_sid_trie_workspace_bytes(int64_t N, int C, int K);
size_t rqb200_sid_trie_scratch_bytes(int64_t N, int C, int K);
int rqb200_sid_trie_build(const int64_t* cached_ids, int64_t N, int C, int K, void* workspace, size_t ws_bytes, void* scratch,
                          size_t scratch_bytes, void* stream);
int rqb200_sid_trie_check(const int64_t* prefix, int64_t row_stride, int64_t P, int l, int C, int K, const void* workspace,
                          unsigned char* valid, void* stream);
int rqb200_sid_trie_beam_select(const int64_t* samples, const float* samp_log_p, const int64_t* generated,
                                const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K,
                                const void* prefix_workspace, int64_t* out_generated, float* out_log_probas, int64_t* out_parent,
                                void* stream);

/* sid_trie_sample_select : the sampling step of the same beam search fused with sid_trie_beam_select, one launch per level h
 *                     (modules/model.py:345-388 after the softmax).  torch.multinomial(p, nc) without replacement is
 *                     topk(p / q, nc) with q = empty_like(p).exponential_(1) from the same generator; given that q in `noise`,
 *                     this call reproduces its samples bit for bit and then selects exactly as sid_trie_beam_select does:
 *   probas, noise    [B*kp, K] fp32, row strides in elements (kp = 1 at h = 0, where generated and log_probas are null)
 *   generated        [B, kp, h] int64, log_probas [B, kp] fp32: the beams entering the level
 *   per row          ratio = probas / noise (IEEE fp32 division), the nc largest ratios in torch.topk's order (descending, NaN
 *                    largest, equal ratios by ascending index) are the samples, samp_log_p = logf(probas[sample])
 *   selection        score = samp_log_p + the parent's log-probability, -inf when the extended prefix is not in the corpus; the
 *                    k best in descending order (ties: lowest candidate index; NaN last) -> out_generated [B, k, h + 1],
 *                    out_log_probas [B, k], out_parent [B*k] = b * kp + beam
 *   samples, samp_log_p  [B*kp, nc], optional (null: not written)
 *   reject           optional int[2], ADDED to (never cleared): [0] rows holding a NaN, +-inf or negative probability, [1] other
 *                    rows whose probabilities are all zero -- the rows torch.multinomial would reject with "probability
 *                    tensor contains either `inf`, `nan` or element < 0" / "invalid multinomial distribution (sum of
 *                    probabilities <= 0)".  Such rows still complete, with unspecified samples in [0, K).
 *   limits           1 <= nc <= K <= 2048, kp * nc <= 1024, k <= 32, h < C <= 8; RQB_ERR_UNSUPPORTED otherwise.
 *                    Deterministic: no result depends on the order of atomics. */
int rqb200_sid_trie_sample_select(const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride,
                                  const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k, int C,
                                  int K, const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                  int64_t* out_parent, int64_t* samples, float* samp_log_p, int* reject, void* stream);
/* sid_trie_sample_select_excluding : the same call with each history's exclusion set (sid_exclusion_build; ex_count null: none).
 *                    After the beam's children are expanded, those that are blocked for its history (level h + 1 of ex_blocked)
 *                    are invalid, exactly like a prefix the corpus lacks.  The noise, samples and samp_log_p are unchanged.
 *                    Needs ex_H > h and ex_M <= 4096. */
int rqb200_sid_trie_sample_select_excluding(const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride,
                                            const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k,
                                            int C, int K, const void* prefix_workspace, int64_t* out_generated,
                                            float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p,
                                            int* reject, const int* ex_pos, const int64_t* ex_blocked, const int* ex_count, int ex_M,
                                            int ex_H, void* stream);
/* sid_trie_sample_select_including : the same call with each history's allow-list (sid_inclusion_build; in_count null: none).
 *                    A beam's children are the keys of level h + 1 of in_keys under its prefix (the prefixes holding an eligible
 *                    item); every other extension is invalid, exactly like a prefix the corpus lacks.  The noise, samples and
 *                    samp_log_p are unchanged.  Needs in_H > h and in_M <= 4096. */
int rqb200_sid_trie_sample_select_including(const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride,
                                            const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k,
                                            int C, int K, const void* prefix_workspace, int64_t* out_generated,
                                            float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p,
                                            int* reject, const int* in_pos, const int64_t* in_keys, const int* in_count, int in_M,
                                            int in_H, void* stream);

/* sid_trie_beam_topk : one level h of the exhaustive (deterministic) constrained beam search, from the head's logits, one launch:
 *   logits           [B*kp, K] fp32, row stride in elements (kp = 1 at h = 0, where generated and log_probas may be null)
 *   generated        [B, kp, h] int64, log_probas [B, kp] fp32: the beams entering the level
 *   per row          lse = m + logf(sum expf(x - m)) in fp32 (m the row maximum, fixed reduction order)
 *   selection        candidate e = beam * K + c of every beam and code scores (x[c] - lse) + log_probas[beam], -inf when
 *                    generated[beam] ++ c is not a corpus prefix or the score is NaN; the k best in descending order (ties:
 *                    lowest e) -> out_generated [B, k, h + 1], out_log_probas [B, k], out_parent [B*k] = b * kp + beam
 *   bad              optional int[1], ADDED to (never cleared): beam rows holding a NaN or +inf logit, or whose logits are all
 *                    -inf.  Such rows still complete; all their candidates score -inf.
 *   limits           K <= 2048, k <= 32, k <= K, kp <= 32, h < C <= 8; RQB_ERR_UNSUPPORTED otherwise.  B = 0 is a no-op.
 *                    Deterministic: no result depends on the order of atomics. */
int rqb200_sid_trie_beam_topk(const float* logits, int64_t logits_stride, const int64_t* generated, const float* log_probas, int B,
                              int kp, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
                              float* out_log_probas, int64_t* out_parent, int* bad, void* stream);
/* sid_trie_beam_topk_excluding : the same call with each history's exclusion set, as sid_trie_sample_select_excluding: a blocked
 *                    extension scores -inf like one the corpus lacks. */
int rqb200_sid_trie_beam_topk_excluding(const float* logits, int64_t logits_stride, const int64_t* generated, const float* log_probas,
                                        int B, int kp, int h, int k, int C, int K, const void* prefix_workspace,
                                        int64_t* out_generated, float* out_log_probas, int64_t* out_parent, int* bad,
                                        const int* ex_pos, const int64_t* ex_blocked, const int* ex_count, int ex_M, int ex_H,
                                        void* stream);
/* sid_trie_beam_topk_including : the same call with each history's allow-list, as sid_trie_sample_select_including: an extension
 *                    to a prefix without an eligible item scores -inf like one the corpus lacks. */
int rqb200_sid_trie_beam_topk_including(const float* logits, int64_t logits_stride, const int64_t* generated, const float* log_probas,
                                        int B, int kp, int h, int k, int C, int K, const void* prefix_workspace,
                                        int64_t* out_generated, float* out_log_probas, int64_t* out_parent, int* bad,
                                        const int* in_pos, const int64_t* in_keys, const int* in_count, int in_M, int in_H,
                                        void* stream);
/* sid_trie_beam_topk_capped : sid_trie_beam_topk with a cap on how many kept beams share a prefix.  A candidate's group is its
 *                    parent's first prefix_len ids.  Walking down the uncapped order (score descending, lowest e first), a
 *                    candidate is kept unless max_per_prefix candidates of its group were kept before it: each group keeps its
 *                    max_per_prefix best, the others score -inf and rank among the -inf fillers by e.  So among a row's kept
 *                    beams with a finite score at most max_per_prefix share a prefix; every kept score has the uncapped bits.
 *   prefix_len       1 <= prefix_len <= h;  max_per_prefix >= 1; RQB_ERR_INVALID otherwise.  max_per_prefix >= k cannot bind
 *                    and runs the uncapped kernel.
 *   filter_mode      0 none, 1 an exclusion, 2 an allow-list: then f_pos .. f_H are the arguments of
 *                    sid_trie_beam_topk_excluding / _including (null / 0 with mode 0).
 *   limits           as sid_trie_beam_topk (no cluster variant). */
int rqb200_sid_trie_beam_topk_capped(const float* logits, int64_t logits_stride, const int64_t* generated, const float* log_probas,
                                     int B, int kp, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
                                     float* out_log_probas, int64_t* out_parent, int* bad, int prefix_len, int max_per_prefix,
                                     int filter_mode, const int* f_pos, const int64_t* f_keys, const int* f_count, int f_M, int f_H,
                                     void* stream);

/* sid_trie_beam_topk_wide : one level of the same exhaustive search for up to 1024 beams per history, on one thread-block
 *                    cluster per history.  Arguments, scores, order, `bad` and results as sid_trie_beam_topk, bit for bit
 *                    wherever both run.
 *   cluster          CTAs per history: 1, 2, 4 or 8, or 0 to let the call choose from B, kp, K and the SM count.  A size whose
 *                    shared memory cannot hold the level or of which no cluster can be resident is RQB_ERR_UNSUPPORTED when
 *                    asked for, skipped when choosing.  No result depends on the size.
 *   limits           K <= 2048, k <= 1024, k <= K, kp <= 1024, h < C <= 8; RQB_ERR_UNSUPPORTED otherwise.  B = 0 is a no-op.
 * _excluding / _including take the filter arguments of sid_trie_beam_topk_excluding / _including after `cluster`. */
int rqb200_sid_trie_beam_topk_wide(const float* logits, int64_t logits_stride, const int64_t* generated, const float* log_probas,
                                   int B, int kp, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
                                   float* out_log_probas, int64_t* out_parent, int* bad, int cluster, void* stream);
int rqb200_sid_trie_beam_topk_wide_excluding(const float* logits, int64_t logits_stride, const int64_t* generated,
                                             const float* log_probas, int B, int kp, int h, int k, int C, int K,
                                             const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                             int64_t* out_parent, int* bad, int cluster, const int* ex_pos, const int64_t* ex_blocked,
                                             const int* ex_count, int ex_M, int ex_H, void* stream);
int rqb200_sid_trie_beam_topk_wide_including(const float* logits, int64_t logits_stride, const int64_t* generated,
                                             const float* log_probas, int B, int kp, int h, int k, int C, int K,
                                             const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                             int64_t* out_parent, int* bad, int cluster, const int* in_pos, const int64_t* in_keys,
                                             const int* in_count, int in_M, int in_H, void* stream);
/* sid_trie_sample_select_wide : one level of the sampled search for up to 1024 beams per history, on one thread-block cluster
 *                    per history.  Arguments, draws, scores, order, `reject` and results as sid_trie_sample_select, bit for bit
 *                    wherever both run; when k > kp * nc the slots past kp * nc repeat candidate 0 with -inf.
 *   workspace        device scratch of sid_trie_sample_select_wide_workspace_bytes(B, kp, nc) bytes (every draw's token and key)
 *   cluster          as sid_trie_beam_topk_wide.
 *   limits           1 <= nc <= 64, nc <= K <= 2048, kp <= 1024, k <= 1024, h < C <= 8; RQB_ERR_UNSUPPORTED otherwise.
 * _excluding / _including take the filter arguments of sid_trie_sample_select_excluding / _including after `cluster`. */
size_t rqb200_sid_trie_sample_select_wide_workspace_bytes(int B, int kp, int nc);
int rqb200_sid_trie_sample_select_wide(const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride,
                                       const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k, int C,
                                       int K, const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                       int64_t* out_parent, int64_t* samples, float* samp_log_p, int* reject, void* workspace,
                                       size_t workspace_bytes, int cluster, void* stream);
int rqb200_sid_trie_sample_select_wide_excluding(const float* probas, int64_t probas_stride, const float* noise,
                                                 int64_t noise_stride, const int64_t* generated, const float* log_probas, int B,
                                                 int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace,
                                                 int64_t* out_generated, float* out_log_probas, int64_t* out_parent,
                                                 int64_t* samples, float* samp_log_p, int* reject, void* workspace,
                                                 size_t workspace_bytes, int cluster, const int* ex_pos, const int64_t* ex_blocked,
                                                 const int* ex_count, int ex_M, int ex_H, void* stream);
int rqb200_sid_trie_sample_select_wide_including(const float* probas, int64_t probas_stride, const float* noise,
                                                 int64_t noise_stride, const int64_t* generated, const float* log_probas, int B,
                                                 int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace,
                                                 int64_t* out_generated, float* out_log_probas, int64_t* out_parent,
                                                 int64_t* samples, float* samp_log_p, int* reject, void* workspace,
                                                 size_t workspace_bytes, int cluster, const int* in_pos, const int64_t* in_keys,
                                                 const int* in_count, int in_M, int in_H, void* stream);
/* sid_trie_sample_select_warped : one level of the sampled search drawn from the head's logits at a temperature and within a
 *                    top-p nucleus (the same kernel as sid_trie_sample_select, in its warped mode).  Per beam row x:
 *                      p_T = expf((x - max x) / temperature) / S, S their fp32 sum; N = {c : p_T[c] >= t}, t the largest p_T
 *                      whose codes at or above it hold at least top_p of the total mass (integer fixed-point sums, 2^-40 units;
 *                      ties at t all in; top_p = 1: every code); the beam draws the min(nc, |N+|) largest p_T / noise over
 *                      N+ = the codes of N with p_T > 0 (equal ratios by ascending code); the other slots are -inf fillers.
 *                    A drawn code scores (x[c] - lse) + log_probas[beam], lse as sid_trie_beam_topk computes it, -inf off the
 *                    trie or blocked by the filter; samp_log_p = x[c] - lse (-inf for a filler).  Selection as
 *                    sid_trie_sample_select.
 *   logits           [B * kp, K] fp32 rows (row stride logits_stride), in place of probas
 *   bad              int32 device counter or null: ADDED the number of beam rows holding a NaN or +inf, or all -inf
 *   temperature      finite, > 0;  top_p in (0, 1]; RQB_ERR_INVALID otherwise
 * _excluding / _including take the filter arguments of sid_trie_sample_select_excluding / _including after top_p; the _wide
 * variants are sid_trie_sample_select_wide's cluster kernel in the same mode (workspace and cluster before temperature). */
int rqb200_sid_trie_sample_select_warped(const float* logits, int64_t logits_stride, const float* noise, int64_t noise_stride,
                                         const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k,
                                         int C, int K, const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                         int64_t* out_parent, int64_t* samples, float* samp_log_p, int* bad, float temperature,
                                         float top_p, void* stream);
int rqb200_sid_trie_sample_select_warped_excluding(const float* logits, int64_t logits_stride, const float* noise,
                                                   int64_t noise_stride, const int64_t* generated, const float* log_probas, int B,
                                                   int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace,
                                                   int64_t* out_generated, float* out_log_probas, int64_t* out_parent,
                                                   int64_t* samples, float* samp_log_p, int* bad, float temperature, float top_p,
                                                   const int* ex_pos, const int64_t* ex_blocked, const int* ex_count, int ex_M,
                                                   int ex_H, void* stream);
int rqb200_sid_trie_sample_select_warped_including(const float* logits, int64_t logits_stride, const float* noise,
                                                   int64_t noise_stride, const int64_t* generated, const float* log_probas, int B,
                                                   int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace,
                                                   int64_t* out_generated, float* out_log_probas, int64_t* out_parent,
                                                   int64_t* samples, float* samp_log_p, int* bad, float temperature, float top_p,
                                                   const int* in_pos, const int64_t* in_keys, const int* in_count, int in_M,
                                                   int in_H, void* stream);
/* sid_trie_sample_select_capped / sid_trie_sample_select_warped_capped : sid_trie_sample_select / _warped with the per-prefix cap
 *                    of sid_trie_beam_topk_capped on the selection, in the candidates' order (score descending, lowest
 *                    beam * nc + slot first).  The draws, samples and samp_log_p do not change.  prefix_len, max_per_prefix
 *                    and the filter arguments as sid_trie_beam_topk_capped; limits as sid_trie_sample_select (no cluster
 *                    variant). */
int rqb200_sid_trie_sample_select_capped(const float* probas, int64_t probas_stride, const float* noise, int64_t noise_stride,
                                         const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k,
                                         int C, int K, const void* prefix_workspace, int64_t* out_generated, float* out_log_probas,
                                         int64_t* out_parent, int64_t* samples, float* samp_log_p, int* reject, int prefix_len,
                                         int max_per_prefix, int filter_mode, const int* f_pos, const int64_t* f_keys,
                                         const int* f_count, int f_M, int f_H, void* stream);
int rqb200_sid_trie_sample_select_warped_capped(const float* logits, int64_t logits_stride, const float* noise,
                                                int64_t noise_stride, const int64_t* generated, const float* log_probas, int B, int kp,
                                                int nc, int h, int k, int C, int K, const void* prefix_workspace,
                                                int64_t* out_generated, float* out_log_probas, int64_t* out_parent, int64_t* samples,
                                                float* samp_log_p, int* bad, float temperature, float top_p, int prefix_len,
                                                int max_per_prefix, int filter_mode, const int* f_pos, const int64_t* f_keys,
                                                const int* f_count, int f_M, int f_H, void* stream);
int rqb200_sid_trie_sample_select_warped_wide(const float* logits, int64_t logits_stride, const float* noise, int64_t noise_stride,
                                              const int64_t* generated, const float* log_probas, int B, int kp, int nc, int h, int k,
                                              int C, int K, const void* prefix_workspace, int64_t* out_generated,
                                              float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p,
                                              int* bad, void* workspace, size_t workspace_bytes, int cluster, float temperature,
                                              float top_p, void* stream);
int rqb200_sid_trie_sample_select_warped_wide_excluding(
    const float* logits, int64_t logits_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* bad, void* workspace,
    size_t workspace_bytes, int cluster, float temperature, float top_p, const int* ex_pos, const int64_t* ex_blocked,
    const int* ex_count, int ex_M, int ex_H, void* stream);
int rqb200_sid_trie_sample_select_warped_wide_including(
    const float* logits, int64_t logits_stride, const float* noise, int64_t noise_stride, const int64_t* generated,
    const float* log_probas, int B, int kp, int nc, int h, int k, int C, int K, const void* prefix_workspace, int64_t* out_generated,
    float* out_log_probas, int64_t* out_parent, int64_t* samples, float* samp_log_p, int* bad, void* workspace,
    size_t workspace_bytes, int cluster, float temperature, float top_p, const int* in_pos, const int64_t* in_keys,
    const int* in_count, int in_M, int in_H, void* stream);

/* The trie's level arrays as plain device arrays (the exact ranking decodes one row per node).
 * sid_trie_counts : counts int32 [C + 1] = the node count of every level (counts[0] = 1, the root); one tiny launch.
 * sid_trie_level  : for level l (1..C) of n_l nodes below n_prev parents: code int32 [n_l] (each node's last id), parent int32
 *                   [n_l] (its node in level l - 1) and, for l < C, child int32 [n_l + 1] (node i's children in level l + 1 are
 *                   child[i] .. child[i + 1] - 1; null when l = C).  n_l and n_prev must be the counts above. */
int rqb200_sid_trie_counts(const void* workspace, int* counts, void* stream);
int rqb200_sid_trie_level(const void* workspace, int C, int l, int n_l, int n_prev, int* code, int* parent, int* child,
                          void* stream);

/* ---- from generated id tuples to corpus items ----
 * Row n of the corpus id table [N, C] is item n; rows with equal tuples are told apart by their dedup rank (the tokeniser's last
 * column: how many earlier rows carry the same tuple).  The item table maps a tuple back to its rows.  A row is retrievable
 * only if all C of its ids are in [0, K); duplicated rows and N = 0 are legal.  Limits: C <= 8, K <= 65536, N < 2^31 - 1.
 * sid_items_build     : stable radix sort of the rows on their packed tuple (the trie build's sort), then one scan over the
 *                       first row of each distinct tuple.  The workspace (sid_items_workspace_bytes: O(N C) bytes, 0 outside the
 *                       limits or when the current device cannot be queried) starts with a header that locates row [N] (row
 *                       ids in sorted order; equal tuples in ascending row order, i.e. dedup rank 0, 1, 2, ...), the U distinct
 *                       tuples' keys and start [U + 1] (tuple u's rows are row[start[u] .. start[u + 1])).  Runs on the stream
 *                       without synchronising the host.
 * sid_items_lookup    : out_item[p] for the tuple ids[p, 0:C] (row stride ids_stride, in elements): its first item, or with
 *                       with_dedup the item of dedup rank d = ids[p, C]; -1 when the tuple holds an id outside [0, K), is not
 *                       in the corpus, or d is outside [0, count).
 * sid_items_retrieve  : generated [B, k, C] int64 (contiguous), log_probas [B, k] fp32 or null -> per history b, in beam order
 *                       (generate returns beams by descending score), the items of every beam whose log-probability is above
 *                       -inf (or log_probas is null) and whose tuple is in the corpus, each beam's in ascending row order
 *                       (dedup rank 0, 1, ...), an item already written for b not repeated (two beams with one tuple), cut off
 *                       at n: out_items [B, n] int64 (-1 pad), out_beam [B, n] int32 (the source beam, -1 pad), out_count [B]
 *                       int32.  C must be the table's C (else no beam resolves).  One CTA per history; deterministic.
 *                       Limits: k <= 1024, n <= 4096, RQB_ERR_UNSUPPORTED otherwise.  B = 0 is a no-op. */
size_t rqb200_sid_items_workspace_bytes(int64_t N, int C, int K);
int rqb200_sid_items_build(const int64_t* cached_ids, int64_t N, int C, int K, void* workspace, size_t ws_bytes, void* stream);
int rqb200_sid_items_lookup(const void* workspace, const int64_t* ids, int64_t ids_stride, int64_t P, int with_dedup,
                            int64_t* out_item /* [P] */, void* stream);
int rqb200_sid_items_retrieve(const void* workspace, const int64_t* generated, const float* log_probas, int B, int k, int C, int n,
                              int64_t* out_items, int* out_beam, int* out_count, void* stream);
/* sid_items_retrieve_excluding : the same call with each history's exclusion set (sid_exclusion_build, on this table): a beam
 *                       counts its tuple's items that are not excluded, in dedup order; an excluded item is never written. */
int rqb200_sid_items_retrieve_excluding(const void* workspace, const int64_t* generated, const float* log_probas, int B, int k, int C,
                                        int n, int64_t* out_items, int* out_beam, int* out_count, const int* ex_pos,
                                        const int64_t* ex_blocked, const int* ex_count, int ex_M, int ex_H, void* stream);
/* sid_exclusion_build : each history's exclusion set, one CTA per history.  items int64 [B, M] (corpus rows; -1 pads, repeats
 *                       allowed; M <= 4096), inv int32 [N] (item -> its position in the table's row array), start int32 [U + 1]
 *                       (sid_items_offsets), leaf_key int64 [U] (the table's U tuples packed K-ary, level 0 most significant,
 *                       ascending), H the tuple length (H * bits(K - 1) <= 62).  Writes
 *                         pos int32 [B, M]          the distinct positions of the retrievable excluded items, ascending (-1 after);
 *                         blocked int64 [B, H, M]   per level l = 1..H the packed keys of the blocked l-prefixes, ascending (-1
 *                                                   after): prefixes holding an excluded item under which every retrievable item
 *                                                   is excluded;
 *                         count int32 [B, H + 2]    [0] the positions, [l] the blocked l-prefixes, [H + 1] the entries outside
 *                                                   [-1, N) (otherwise ignored).
 *                       Unretrievable rows (positions from start[U] on) are ignored.  Plain stores: the output is a function
 *                       of the input.  B = 0 is a no-op. */
int rqb200_sid_exclusion_build(const int64_t* items, int B, int M, int64_t N, const int* inv, const int* start,
                               const int64_t* leaf_key, int U, int H, int K, int* pos, int64_t* blocked, int* count, void* stream);
/* sid_items_retrieve_including : the same call with each history's allow-list (sid_inclusion_build, on this table): a beam counts
 *                       its tuple's eligible items, in dedup order; no other item is written. */
int rqb200_sid_items_retrieve_including(const void* workspace, const int64_t* generated, const float* log_probas, int B, int k, int C,
                                        int n, int64_t* out_items, int* out_beam, int* out_count, const int* in_pos,
                                        const int64_t* in_keys, const int* in_count, int in_M, int in_H, void* stream);
/* sid_inclusion_build : each history's allow-list, one CTA per history, with the arguments of sid_exclusion_build plus an optional
 *                       exclusion of the same histories (its arrays; ex_count null: none), which is folded in.  items are the
 *                       allowed corpus rows (-1 pads, repeats allowed, M <= 4096).  An item is eligible when it is allowed,
 *                       retrievable and not excluded.  Writes
 *                         pos int32 [B, M]          the distinct positions of the eligible items, ascending (-1 after);
 *                         keys int64 [B, H, M]      per level l = 1..H the packed keys of the distinct l-prefixes of the eligible
 *                                                   items (the valid l-prefixes), ascending (-1 after);
 *                         count int32 [B, H + 2]    [0] the positions, [l] the valid l-prefixes, [H + 1] the entries of items
 *                                                   outside [-1, N) (otherwise ignored).
 *                       Plain stores: the output is a function of the input.  B = 0 is a no-op. */
int rqb200_sid_inclusion_build(const int64_t* items, int B, int M, int64_t N, const int* inv, const int* start,
                               const int64_t* leaf_key, int U, int H, int K, int* pos, int64_t* keys, int* count,
                               const int* ex_pos, const int64_t* ex_blocked, const int* ex_count, int ex_M, int ex_H, void* stream);
/* sid_items_offsets   : byte offsets of row (int32 [N]) and start (int32 [N + 1]) in the item table's workspace; arithmetic only.
 *                       RQB_ERR_UNSUPPORTED outside the table's limits. */
int rqb200_sid_items_offsets(int64_t N, int C, int K, size_t* row, size_t* start);

/* sid_topk_rank_hist  : evaluate/metrics.py's TopKAccumulator rule, accumulated on the device.  Row b's rank is its first
 *                       candidate cand[b, j, 0:D] equal to actual[b, 0:D] in all D columns (`.all(-1).max(-1)`); hist[rank] += 1,
 *                       or hist[k] += 1 when none matches.  hist is int64 [k + 1], ADDED to (never cleared), so batches
 *                       accumulate exactly; NDCG = sum_r hist[r] / log2(r + 2) and h@j = sum_{r<j} hist[r] follow from it.
 *                       item_mode: a value -1 (padding, an unresolvable item) never matches; otherwise every input keeps the
 *                       reference's rule.  actual row stride a_stride >= D, cand [B, k, D] with history stride c_stride >= k D
 *                       (elements).  B = 0 is a no-op. */
int rqb200_sid_topk_rank_hist(const int64_t* actual, int64_t a_stride, const int64_t* cand, int64_t c_stride, int B, int k, int D,
                              int item_mode, int64_t* hist, void* stream);
/* sid_rank_hist       : hist[rank[b]] += 1 for an exact rank in [0, k), hist[k] += 1 otherwise (-1: the item is not ranked).
 *                       rank int64 [B], hist int64 [k + 1], ADDED to.  B = 0 is a no-op. */
int rqb200_sid_rank_hist(const int64_t* rank, int B, int64_t k, int64_t* hist, void* stream);

/* ---- exact ranking of every corpus item (modules/model.py rank_sem_ids / rank_items), csrc/t5rank.cu ----
 * t5rank_cross_attention : T5 cross-attention (no 1/sqrt(d) scaling, fp32 softmax) of Q queries per history: q [B * Q, inner] (row
 *                          stride ldq; history b's queries are rows b * Q ..), keys / values of history b the rows offsets[b] ..
 *                          offsets[b + 1] - 1 of k / v (row stride ldkv; offsets int32 [B + 1], absolute rows), score q . k +
 *                          key_mask[row] (fp32 [rows]: 0, or -FLT_MAX to mask; null: 0).  out [B * Q, inner] (row stride ldo);
 *                          a history without keys gets zeros.  Limits: B, heads <= 65535.
 * t5rank_cross_attention_tc : the same call with S = Q K^T and P V as wgmma m64n64k8 TF32 (operands rounded to TF32, fp32
 *                          accumulate), softmax and mask in fp32; q, k, v 16-byte aligned with row strides a multiple of 4.
 * t5rank_children        : logits [R, K] (row stride ld) of R = B * n_h node rows of one trie level (row b * n_h + i); per row
 *                          lse = m + logf(sum expf(x - m)) exactly as sid_trie_beam_topk, and for every child j of node i (child
 *                          int32 [n_h + 1]: child[i] <= j < child[i + 1]) out[b * n_next + j] = (x[code[j]] - lse) + parent[r]
 *                          (parent fp32 [R], null: 0; code int32 [n_next]).  A row holding a NaN or +inf logit, or all -inf, adds 1
 *                          to bad (int32 [1], optional) and gives its children NaN.
 * t5rank_select          : one CTA per history over its U leaf scores (scores fp32 [B, U], leaf u = item-table tuple u; row / start
 *                          the item table's arrays, sid_items_offsets).  Order: score descending, then leaf ascending, NaN last;
 *                          each leaf's items in dedup order.  out_items int64 [B, n] / out_scores fp32 [B, n] (the item's leaf
 *                          score): the first n items, -1 / -inf past the corpus.  out_rank int64 [B]: the position in that order of
 *                          item t_dedup[b] of leaf t_leaf[b] (int64 [B] each), -1 when t_leaf is outside [0, U) or the dedup rank
 *                          outside the leaf's items.  n <= 1024 (RQB_ERR_UNSUPPORTED).  No global atomics: deterministic. */
int rqb200_t5rank_cross_attention(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv, const int* offsets,
                                  const float* key_mask, int B, int Q, int heads, float* out, int64_t ldo, void* stream);
int rqb200_t5rank_cross_attention_tc(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv, const int* offsets,
                                     const float* key_mask, int B, int Q, int heads, float* out, int64_t ldo, void* stream);
int rqb200_t5rank_children(const float* logits, int64_t ld, int R, int K, int n_h, const float* parent, const int* child,
                           const int* code, int n_next, float* out, int* bad, void* stream);
int rqb200_t5rank_select(const float* scores, int B, int U, const int* row, const int* start, const int64_t* t_leaf,
                         const int64_t* t_dedup, int n, int64_t* out_items, float* out_scores, int64_t* out_rank, void* stream);
/* t5rank_select_excluding : the same call with each history's exclusion set (sid_exclusion_build): excluded items are skipped,
 *                          leaves whose items are all excluded take no part, out_rank is the target's position among the items
 *                          that are not excluded (-1 when it is excluded). */
int rqb200_t5rank_select_excluding(const float* scores, int B, int U, const int* row, const int* start, const int64_t* t_leaf,
                                   const int64_t* t_dedup, int n, int64_t* out_items, float* out_scores, int64_t* out_rank,
                                   const int* ex_pos, const int64_t* ex_blocked, const int* ex_count, int ex_M, int ex_H,
                                   void* stream);
/* t5score_trie_build     : the trie of each history's own candidate tuples (modules/model.py score_sem_ids / score_items), one CTA per
 *                          history.  ids int64 [B, C, H] (candidate c of history b: ids[(b * C + c) * H ..]); a tuple holding an id
 *                          outside [0, K) is invalid.  Per history b and level l = 1..H (the distinct l-prefixes of its valid tuples,
 *                          in lexicographic order): counts int32 [B, H] (entry l - 1: the node count n_l), code / parent int32
 *                          [B, H, C] (entry (l - 1, i): node i's last id and its node in level l - 1; 0 and 0 for i >= n_l), child
 *                          int32 [B, H, C + 1] (entry (l, i) for l = 0..H - 1: node i's children in level l + 1 are child[l][i] ..
 *                          child[l][i + 1] - 1; n_{l + 1} for i >= n_l), leaf int32 [B, C] (each candidate's node in level H, -1 when
 *                          invalid; equal tuples share it).  C <= 4096, H <= 8, H * bits(K - 1) <= 62 (RQB_ERR_UNSUPPORTED).  No
 *                          atomics: the output is a function of the input. */
int rqb200_t5score_trie_build(const int64_t* ids, int B, int C, int H, int K, int* counts, int* code, int* parent, int* child,
                              int* leaf, void* stream);

/* ---- exact top-k search (modules/model.py generate(search="exact"), FusedT5Exact), csrc/t5rank.cu ----
 * t5rank_cross_attention_ragged : t5rank_cross_attention over a ragged level: T query tiles, tile t = tiles[3 t ..] (int32:
 *                          history b, first query row, query count <= 64), each over history b's keys; a query's arithmetic is
 *                          that of the uniform fp32 kernel.  Limits: heads <= 65535.
 * t5exact_frontier       : one CTA per history b of Bc over its scored children, nodes of trie level l (1 <= l < 8): entries
 *                          coff[b] .. coff[b + 1] - 1 of sc / cnode / ccode / cpar (fp32 score, node id, last code, parent row), or
 *                          with cnode null (l = 1, the root's children) entries b n_root .. of sc, child i being node i (code
 *                          ccode[i], parent row b).  A child is kept when sc >= tau[b] (NaN never) and the filter does not block its
 *                          prefix key pkey[parent] K + code (pkey int64 [rows], null at l = 1; needed with a filter).  Count pass
 *                          (counts int32 [3, Bc], offs null): per history the kept rows, their children (lchild: the child ranges of
 *                          level l, int32 [n_l + 1]) and their 64-query tiles.  Write pass (offs int32 [3, Bc + 1], the exclusive
 *                          scans of counts, counts null): kept row r (trie order, history b's at offs[0][b] ..) gets row_code /
 *                          row_par int64, row_score fp32, row_key int64 (with a filter), row_node int32; tiles int32 [T, 3] for
 *                          t5rank_cross_attention_ragged; nrng int32 [R + 1] the rows' child ranges (global, for t5rank_children
 *                          as one group), and per child g: nnode (node of level l + 1), ncode (lcode_next[node]), npar (row).
 *                          b0: the chunk's first history in the filter.  Plain stores: the output is a function of the input.
 * t5exact_select         : one CTA per history b over its leaf candidates (coff / cnode / n_root as t5exact_frontier's children,
 *                          cnode the leaf ids; max_u the largest count): the w best by (score descending, leaf ascending), NaN and
 *                          filter-blocked leaves (level H keys leaf_key[leaf], int64 [U]; needed with a filter) left out.  out_gen
 *                          int64 [Bc, w, H] each chosen leaf's tuple along its path (codes / parents: host arrays of H + 1 device
 *                          pointers, entry l = SidTrieLevels.code[l] / parent[l]), out_lp fp32 [Bc, w] its score; -1 / -inf past
 *                          the valid candidates.  w <= 1024, H <= 8 (RQB_ERR_UNSUPPORTED).  No global atomics.
 * _excluding / _including take an exclusion set (sid_exclusion_build) / an allow-list (sid_inclusion_build) of the whole batch
 * (history b0 + b) after the other arguments, as the search kernels. */
int rqb200_t5rank_cross_attention_ragged(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv, const int* offsets,
                                         const float* key_mask, const int* tiles, int T, int heads, float* out, int64_t ldo,
                                         void* stream);
int rqb200_t5exact_frontier(const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode, const int* cpar,
                            const int64_t* pkey, const float* tau, int Bc, int K, int l, const int* lchild, const int* lcode_next,
                            int b0, int* counts, const int* offs, int64_t* row_code, int64_t* row_par, float* row_score,
                            int64_t* row_key, int* row_node, int* tiles, int* nrng, int* nnode, int* ncode, int* npar, void* stream);
int rqb200_t5exact_frontier_excluding(const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode,
                                      const int* cpar, const int64_t* pkey, const float* tau, int Bc, int K, int l, const int* lchild,
                                      const int* lcode_next, int b0, int* counts, const int* offs, int64_t* row_code,
                                      int64_t* row_par, float* row_score, int64_t* row_key, int* row_node, int* tiles, int* nrng,
                                      int* nnode, int* ncode, int* npar, const int* ex_pos, const int64_t* ex_blocked,
                                      const int* ex_count, int ex_M, int ex_H, void* stream);
int rqb200_t5exact_frontier_including(const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode,
                                      const int* cpar, const int64_t* pkey, const float* tau, int Bc, int K, int l, const int* lchild,
                                      const int* lcode_next, int b0, int* counts, const int* offs, int64_t* row_code,
                                      int64_t* row_par, float* row_score, int64_t* row_key, int* row_node, int* tiles, int* nrng,
                                      int* nnode, int* ncode, int* npar, const int* in_pos, const int64_t* in_keys,
                                      const int* in_count, int in_M, int in_H, void* stream);
int rqb200_t5exact_select(const float* sc, const int* coff, int n_root, const int* cnode, int max_u, const int64_t* leaf_key,
                          const void* const* codes, const void* const* parents, int Bc, int H, int w, int b0, int64_t* out_gen,
                          float* out_lp, void* stream);
int rqb200_t5exact_select_excluding(const float* sc, const int* coff, int n_root, const int* cnode, int max_u,
                                    const int64_t* leaf_key, const void* const* codes, const void* const* parents, int Bc, int H,
                                    int w, int b0, int64_t* out_gen, float* out_lp, const int* ex_pos, const int64_t* ex_blocked,
                                    const int* ex_count, int ex_M, int ex_H, void* stream);
int rqb200_t5exact_select_including(const float* sc, const int* coff, int n_root, const int* cnode, int max_u,
                                    const int64_t* leaf_key, const void* const* codes, const void* const* parents, int Bc, int H,
                                    int w, int b0, int64_t* out_gen, float* out_lp, const int* in_pos, const int64_t* in_keys,
                                    const int* in_count, int in_M, int in_H, void* stream);

/* ---- one step of the generative-retrieval model's T5 decoder (modules/model.py, generate(decoder="fused")), csrc/t5dec.cu ----
 * HF T5 numerics in eval mode: attention without 1/sqrt(d) scaling, fp32 softmax, d_kv = 64 per head (inner = heads * 64).
 * The GEMMs around these calls are the caller's.  fp32 throughout; strides in elements.
 * t5dec_cross_attention : attention over the encoder output with keys/values stored ONCE per history.  q [B * nq, inner] (row
 *                         stride ldq; rows b * nq .. b * nq + nq - 1 belong to history b), k / v [B * S, inner] (row stride ldkv:
 *                         key s of history b is row b * S + s), mask [B, S] or null (a key whose mask is 0 gets -FLT_MAX added,
 *                         torch.finfo(float32).min as in HF's eager mask), out [B * nq, inner] (row stride ldo).  One CTA per
 *                         (head, history, group of 32 queries) reads the history's keys/values once for its queries; a query's
 *                         result does not depend on nq; any S >= 1.
 *                         Limits: nq <= 65535 * 32, B <= 65535 (RQB_ERR_UNSUPPORTED).
 * t5dec_self_attention  : the causal self-attention of query position h (< H <= 8) for R beam rows.  qkv [R, 3 inner] (q | k | v,
 *                         row stride ldqkv).  cache_k / cache_v hold slot j (position j) of row x at [j * slot_stride + x * inner];
 *                         the row's own k / v are written to slot h.  Earlier positions j < h of row r are read from row
 *                         anc[r, j] of slot j, anc = int32 [rows, H]: anc = anc_in when parent is null; with parent (int64 [R], the
 *                         previous level's row of each beam) anc[r, j] = anc_in[parent[r], j] for j < h - 1 and anc[r, h - 1] =
 *                         parent[r], and this call writes it to anc_out (which must not alias anc_in).  bias [heads, H, H] is added
 *                         to the score of (query h, key j).  out [R, inner] (row stride ldo).
 * t5dec_add_norm        : one sublayer boundary, one warp per row of x [R, D] (contiguous, updated in place):
 *                         emb != null : x[r] = emb[ids[r * ids_stride] + id_offset] (row 0 for all r when ids is null; an id outside
 *                                       [0, n_emb) gives a NaN row) -- the step's input embedding;
 *                         else        : x[r] += delta[r] (row stride ld_delta; null: x unchanged);
 *                         then out[r] = weight * (x[r] * rsqrt(mean(x[r]^2) + eps)) (T5LayerNorm), out [R, D] contiguous. */
int rqb200_t5dec_cross_attention(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv, const float* mask, int B,
                                 int nq, int S, int heads, float* out, int64_t ldo, void* stream);
int rqb200_t5dec_self_attention(const float* qkv, int64_t ldqkv, float* cache_k, float* cache_v, int64_t slot_stride,
                                const float* bias, const int* anc_in, const int64_t* parent, int* anc_out, int R, int heads, int h,
                                int H, float* out, int64_t ldo, void* stream);
int rqb200_t5dec_add_norm(float* x, const float* delta, int64_t ld_delta, const float* emb, const int64_t* ids, int64_t ids_stride,
                          int64_t id_offset, int64_t n_emb, const float* weight, int R, int D, float eps, float* out, void* stream);

/* ---- device-counted launches: the decoder level of a CUDA-graph replay whose row count exists only on the device
 * (modules/model.py FusedT5Exact(capacity=True)) ----
 * Each call takes the host-counted call's arguments, with its row (or tile) count as a CAPACITY that sizes the grid and the
 * buffers, and a device count: rows (tiles) below min(*live, capacity) get the host-counted call's bits at that count, and the
 * CTAs / warps past it exit without writing.  The host-counted entry points are unchanged.
 *   f32_to_split_image_counted : row-major operands only; rows = capacity (the image layout), *live_rows the source rows.
 *   gemm_split_counted         : M = capacity (of the A image), *live_m the rows written.
 *   t5dec_self_attention_counted / t5dec_add_norm_counted : R = capacity, *live_r the rows (ancestor advance and embedding
 *                                gather included).
 *   t5rank_cross_attention_ragged_counted : T = capacity, *live_t the tiles.
 *   t5rank_children_counted    : one group of R = capacity rows (n_h = R), live[0] the rows, live[1] the children (<= n_next, the
 *                                capacity of out / code).
 *   t5exact_frontier_capacity[_excluding/_including] : the write pass of t5exact_frontier with outputs of r_cap rows, c_cap children
 *                                and t_cap tiles, the totals offs[., Bc] read on the device.  When they fit it writes the write
 *                                pass's outputs, live int32 [3] = (R, C, T) and noff int32 [Bc + 1] = offs[1] (the children's
 *                                offsets for the next level).  When a total exceeds its capacity it writes no row, sets live and
 *                                noff to 0 and *overflow = 1 (never cleared here), so the next level's launches find no rows. */
int rqb200_f32_to_split_image_counted(const float* x, int64_t ldx, int rows, int K, const int* live_rows, void* image, void* stream);
int rqb200_gemm_split_counted(const void* a_image, const void* b_image, int M, int N, int K, int relu, const float* mask, int64_t ldm,
                              const int* live_m, float* out, int64_t ldo, void* stream);
int rqb200_t5dec_self_attention_counted(const float* qkv, int64_t ldqkv, float* cache_k, float* cache_v, int64_t slot_stride,
                                        const float* bias, const int* anc_in, const int64_t* parent, int* anc_out, int R,
                                        const int* live_r, int heads, int h, int H, float* out, int64_t ldo, void* stream);
int rqb200_t5dec_add_norm_counted(float* x, const float* delta, int64_t ld_delta, const float* emb, const int64_t* ids,
                                  int64_t ids_stride, int64_t id_offset, int64_t n_emb, const float* weight, int R, const int* live_r,
                                  int D, float eps, float* out, void* stream);
int rqb200_t5rank_cross_attention_ragged_counted(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv,
                                                 const int* offsets, const float* key_mask, const int* tiles, int T, const int* live_t,
                                                 int heads, float* out, int64_t ldo, void* stream);
int rqb200_t5rank_children_counted(const float* logits, int64_t ld, int R, int K, const float* parent, const int* child,
                                   const int* code, int n_next, const int* live, float* out, int* bad, void* stream);
int rqb200_t5exact_frontier_capacity(const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode, const int* cpar,
                                     const int64_t* pkey, const float* tau, int Bc, int K, int l, const int* lchild,
                                     const int* lcode_next, int b0, const int* offs, int64_t* row_code, int64_t* row_par,
                                     float* row_score, int64_t* row_key, int* row_node, int* tiles, int* nrng, int* nnode, int* ncode,
                                     int* npar, int r_cap, int c_cap, int t_cap, int* live, int* overflow, int* noff, void* stream);
int rqb200_t5exact_frontier_capacity_excluding(const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode,
                                               const int* cpar, const int64_t* pkey, const float* tau, int Bc, int K, int l,
                                               const int* lchild, const int* lcode_next, int b0, const int* offs, int64_t* row_code,
                                               int64_t* row_par, float* row_score, int64_t* row_key, int* row_node, int* tiles,
                                               int* nrng, int* nnode, int* ncode, int* npar, int r_cap, int c_cap, int t_cap,
                                               int* live, int* overflow, int* noff, const int* ex_pos, const int64_t* ex_blocked,
                                               const int* ex_count, int ex_M, int ex_H, void* stream);
int rqb200_t5exact_frontier_capacity_including(const float* sc, const int* coff, int n_root, const int* cnode, const int* ccode,
                                               const int* cpar, const int64_t* pkey, const float* tau, int Bc, int K, int l,
                                               const int* lchild, const int* lcode_next, int b0, const int* offs, int64_t* row_code,
                                               int64_t* row_par, float* row_score, int64_t* row_key, int* row_node, int* tiles,
                                               int* nrng, int* nnode, int* ncode, int* npar, int r_cap, int c_cap, int t_cap,
                                               int* live, int* overflow, int* noff, const int* in_pos, const int64_t* in_keys,
                                               const int* in_count, int in_M, int in_H, void* stream);

/* ---- the generative-retrieval model's T5 encoder pass over kept tokens only (modules/model.py, generate(encoder="fused")),
 * csrc/t5enc.cu ----
 * The encoder input of a history of n = items * H ids (mask [B, n] fp32, ids [B, n] int64) has S = user + items * (H + sep)
 * positions: the user row (user = 1), then per item its H ids and, with sep = 1, a separator carrying the mask of the item's last
 * id.  A position is KEPT when its mask is nonzero (the user row always is); a history with no kept position keeps all S, and its
 * keys then get -FLT_MAX added (HF's eager mask: the softmax averages every position).  Kept rows are packed history by history
 * in position order; fp32 throughout, d_kv = 64 per head, sublayer boundaries are rqb200_t5dec_add_norm, GEMMs the caller's.
 * t5enc_offsets  : offsets int32 [B + 1] (history b owns packed rows offsets[b] .. offsets[b + 1] - 1; offsets[B] = N, the
 *                  packed row count) and key_mask fp32 [B] (0, or -FLT_MAX for a history without an unmasked position).  One CTA.
 * t5enc_assemble : src int32 [N] = b * S + p of every packed row, slot int32 [B * S] = its packed row or -1 (dropped), and per
 *                  packed row x = the input row -- user_table[remainder(user_ids[b * user_stride], n_users)] (user_table and
 *                  user_ids both null: no user row), item_table[(ids[b, c] + (c % H) * K) * mask[b, c]] (an id outside
 *                  [0, n_items) gives a NaN row), or sep_row (null: sep = 0) -- and out = T5LayerNorm(x) * weight; x, out [N, D].
 * t5enc_assemble_capacity: t5enc_assemble at a fixed capacity of B * S rows, for a caller that cannot read N (a CUDA-graph
 *                  capture): x, out [B * S, D] and src [B * S]; rows 0 .. N - 1 as t5enc_assemble writes them, rows N .. B * S - 1
 *                  x = out = 0 and src = -1.  No attention kernel reads or writes a row past N, and rqb200_t5dec_add_norm keeps a zero
 *                  row zero, so those rows stay zero through the pass when the attention output's rows past N are zeros.
 * t5enc_attention: bidirectional self-attention among each history's packed rows.  qkv [N, 3 inner] (q | k | v, row stride
 *                  ldqkv, a multiple of 4, 16-byte aligned), rel [heads, 2S - 1]: the score of query position i and key position
 *                  j is q . k + (rel[n, j - i + S - 1] + key_mask[b]), no 1/sqrt(d) scaling, fp32 softmax.  out [N, inner] (row
 *                  stride ldo, a multiple of 4, 16-byte aligned).  Any S.
 * t5enc_scatter  : out[r] = rows[slot[r]] for r < n_out (= B * S), zeros where slot[r] = -1; rows [N, D], out [n_out, D]. */
int rqb200_t5enc_offsets(const float* mask, int B, int n, int H, int sep, int user, int* offsets, float* key_mask, void* stream);
int rqb200_t5enc_assemble(const float* mask, const int64_t* ids, int64_t ids_stride, const int64_t* user_ids, int64_t user_stride,
                          const float* item_table, int64_t n_items, const float* sep_row, const float* user_table, int64_t n_users,
                          int64_t K, int B, int n, int H, int D, const int* offsets, const float* weight, float eps, float* x,
                          float* out, int* src, int* slot, void* stream);
int rqb200_t5enc_assemble_capacity(const float* mask, const int64_t* ids, int64_t ids_stride, const int64_t* user_ids,
                                   int64_t user_stride, const float* item_table, int64_t n_items, const float* sep_row,
                                   const float* user_table, int64_t n_users, int64_t K, int B, int n, int H, int D,
                                   const int* offsets, const float* weight, float eps, float* x, float* out, int* src, int* slot,
                                   void* stream);
int rqb200_t5enc_attention(const float* qkv, int64_t ldqkv, const int* src, const int* offsets, const float* key_mask,
                           const float* rel, int B, int S, int heads, float* out, int64_t ldo, void* stream);
int rqb200_t5enc_scatter(const float* rows, const int* slot, int64_t n_out, int D, float* out, void* stream);

/* ---- training the encoder pass over kept tokens (modules/model.py, forward(encoder="fused")), csrc/t5enc.cu ----
 * Shapes and packing as above.  Attention-weight dropout with probability p (0 <= p < 1) keeps the weight of (history b, head n,
 * query position i, key position j) when the first word of Philox4x32-10(counter {j, i, n, b}, key {seed lo, seed hi}) is at least
 * floor(p * 2^32); seed is int64 [1] in device memory.  Kept weights are scaled by 1 / (1 - p).
 * t5enc_attention_train   : t5enc_attention's output with that dropout, out = sum_j (P_ij keep_ij / (1 - p)) v_j, plus lse [N, heads]
 *                           = (m - key_mask[b]) + log l, the log-sum-exp of the row's scores less key_mask (l the undropped sum).
 * t5enc_attention_backward: from out (the forward's), dout [N, inner] and lse: dS = P (dP keep / (1 - p) - D) with
 *                           D_i = dout_i . out_i written to delta [N, heads]; dqkv [N, 3 inner] (row stride ldd: dQ | dK | dV, every
 *                           column written) and drel_part [B, t5enc_attention_backward_tiles(S), heads, 2S - 1], partial sums of
 *                           d rel whose sum over the first two axes is d rel.  Two launches, no atomics: bit-reproducible.
 *                           S <= 5120 (one shared-memory bin array of 2S - 1 floats per warp).
 * t5enc_dropout_keep      : keep uint8 [B, heads, S, S] (0 / 1), the bits above for every position pair.
 * t5enc_add_norm_fwd      : one warp per row: x_out = x + delta (delta null: x), out = weight * (x_out * inv), inv_rms [R] = inv =
 *                           rsqrt(mean(x_out^2) + eps); x, x_out, out [R, D] contiguous.
 * t5enc_add_norm_bwd      : from d_out [R, D] and d_res [R, D] (the gradient reaching x_out directly; null: 0): dx = d_x_out [R, D]
 *                           (also the gradient of delta) and dw_part [t5enc_add_norm_bwd_parts(R), D], partial sums of d weight in
 *                           a fixed order.  D <= 5120. */
int rqb200_t5enc_attention_train(const float* qkv, int64_t ldqkv, const int* src, const int* offsets, const float* key_mask,
                                 const float* rel, int B, int S, int heads, const int64_t* seed, float p, float* out, int64_t ldo,
                                 float* lse, void* stream);
int rqb200_t5enc_attention_backward_tiles(int S);
int rqb200_t5enc_attention_backward(const float* qkv, int64_t ldqkv, const float* out, int64_t ldo, const float* dout, int64_t lddo,
                                    const float* lse, const int* src, const int* offsets, const float* key_mask, const float* rel,
                                    int B, int S, int heads, const int64_t* seed, float p, float* delta, float* dqkv, int64_t ldd,
                                    float* drel_part, void* stream);
int rqb200_t5enc_dropout_keep(const int64_t* seed, float p, int B, int heads, int S, uint8_t* keep, void* stream);
int rqb200_t5enc_add_norm_fwd(const float* x, const float* delta, int64_t ld_delta, const float* weight, int R, int D, float eps,
                              float* x_out, float* out, float* inv_rms, void* stream);
int rqb200_t5enc_add_norm_bwd_parts(int R);
int rqb200_t5enc_add_norm_bwd(const float* d_out, const float* d_res, const float* x_out, const float* inv_rms, const float* weight,
                              int R, int D, float* dx, float* dw_part, void* stream);

/* ---- TF32 tensor-core encoder self-attention (encoder_attention="tf32"), csrc/t5enc_tc.cu ----
 * The entry points above with the same arguments, layouts, dropout bits and outputs, whose products (scores, P.V, dP and the
 * gradient products) run as wgmma TF32 with fp32 accumulation, operands rounded to TF32.  Softmax, bias, mask and dropout are fp32.
 * t5enc_attention_tc_backward's drel_part is [B, t5enc_attention_tc_backward_tiles(S), heads, 2S - 1]; two launches, no atomics,
 * bit-reproducible; S <= 8336 (two shared-memory bin arrays of 2S - 1 floats). */
int rqb200_t5enc_attention_tc(const float* qkv, int64_t ldqkv, const int* src, const int* offsets, const float* key_mask,
                              const float* rel, int B, int S, int heads, float* out, int64_t ldo, void* stream);
int rqb200_t5enc_attention_tc_train(const float* qkv, int64_t ldqkv, const int* src, const int* offsets, const float* key_mask,
                                    const float* rel, int B, int S, int heads, const int64_t* seed, float p, float* out, int64_t ldo,
                                    float* lse, void* stream);
int rqb200_t5enc_attention_tc_backward_tiles(int S);
int rqb200_t5enc_attention_tc_backward(const float* qkv, int64_t ldqkv, const float* out, int64_t ldo, const float* dout,
                                       int64_t lddo, const float* lse, const int* src, const int* offsets, const float* key_mask,
                                       const float* rel, int B, int S, int heads, const int64_t* seed, float p, float* delta,
                                       float* dqkv, int64_t ldd, float* drel_part, void* stream);

/* ---- training the decoder pass (modules/model.py, forward(decoder="fused")), csrc/t5dec.cu ----
 * T (<= 8, else RQB_ERR_UNSUPPORTED) decoder positions per history: row b * T + t of q / qkv / out / dout holds position t of
 * history b; inner = heads * 64, fp32, strides in elements, no 1/sqrt(d) scaling.  Attention-weight dropout as the encoder's:
 * the weight of (history b, head n, query position t, key position j) is kept when the first word of Philox4x32-10(counter
 * {j, t, n, b}, key {seed lo, seed hi}) is at least floor(p * 2^32), kept weights scaled by 1 / (1 - p); seed int64 [1] in device
 * memory.  No atomics: the backwards are bit-reproducible.
 * t5dec_self_attention_train   : causal self-attention, qkv [B * T, 3 inner] (q | k | v), rel [heads, 2T - 1] (the bias of key j
 *                                for query t is rel[n, j - t + T - 1]); keys j > t get weight 0.  out [B * T, inner], lse
 *                                [B * T, heads] = m + log l of the undropped scores.
 * t5dec_self_attention_backward: from out (the forward's), dout and lse: dqkv [B * T, 3 inner] (dQ | dK | dV) and drel_part
 *                                [B, heads, 2T - 1], partial sums of d rel whose sum over the first axis is d rel.
 * t5dec_cross_attention_train  : attention of q [B * T, inner] over key rows offsets[b] .. offsets[b + 1] - 1 (int32 [B + 1]) of k / v
 *                                (row stride ldkv), score q . k + key_mask[row] (key_mask fp32 [rows]: 0, or -FLT_MAX to mask).
 *                                The key's position j in the dropout counter is src[row] - b * S (src int32 [rows], the packed
 *                                encoder's b * S + p) or, with src null, row - offsets[b].  out [B * T, inner], lse [B * T, heads] =
 *                                (m - base) + log l with base the history's largest key_mask (finite when every key is masked).  A
 *                                history without keys gets zeros.
 * t5dec_cross_attention_backward: from out, dout and lse: dq [B * T, inner] (row stride lddq) and dk / dv (row stride lddkv, the rows
 *                                of k / v; rows no history owns are not written). */
int rqb200_t5dec_self_attention_train(const float* qkv, int64_t ldqkv, const float* rel, int B, int T, int heads, const int64_t* seed,
                                      float p, float* out, int64_t ldo, float* lse, void* stream);
int rqb200_t5dec_self_attention_backward(const float* qkv, int64_t ldqkv, const float* out, int64_t ldo, const float* dout,
                                         int64_t lddo, const float* lse, const float* rel, int B, int T, int heads,
                                         const int64_t* seed, float p, float* dqkv, int64_t ldd, float* drel_part, void* stream);
int rqb200_t5dec_cross_attention_train(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv, const int* offsets,
                                       const float* key_mask, const int* src, int B, int S, int T, int heads, const int64_t* seed,
                                       float p, float* out, int64_t ldo, float* lse, void* stream);
int rqb200_t5dec_cross_attention_backward(const float* q, int64_t ldq, const float* k, const float* v, int64_t ldkv, const float* out,
                                          int64_t ldo, const float* dout, int64_t lddo, const float* lse, const int* offsets,
                                          const float* key_mask, const int* src, int B, int S, int T, int heads,
                                          const int64_t* seed, float p, float* dq, int64_t lddq, float* dk, float* dv, int64_t lddkv,
                                          void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RQB200_H */
