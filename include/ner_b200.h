/*
 * ner_b200.h — C-ABI of libner_b200.so: the sm_90a kernels behind the
 * bert_bilstm_crf hot path of DSXiangLi/ChineseNER.
 *
 * Every entry point mirrors one reference call site (cited per function,
 * paths relative to the reference repo).  Conventions:
 *   - all pointers are BORROWED DEVICE pointers (row-major, contiguous) unless
 *     the parameter name ends in `_host`;
 *   - the library never allocates user-visible memory: workspaces are
 *     caller-provided and sized by the matching *_workspace_bytes();
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*),
 *     stateless and re-entrant; no internal synchronisation;
 *   - return value: NER_OK (0) or a negative status; ner_strerror() names it.
 *     No C++ exception crosses this boundary.
 */
#ifndef NER_B200_H_
#define NER_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NER_OK 0
#define NER_ERR_INVALID_ARG (-1)   /* null pointer, negative size, bad enum */
#define NER_ERR_UNSUPPORTED (-2)   /* e.g. K > 32 tags, H not supported */
#define NER_ERR_WORKSPACE (-3)     /* workspace too small / missing */
#define NER_ERR_NO_DRIVER (-4)     /* driver entry point (TMA encode) not found */
#define NER_ERR_CUDA_BASE (-1000)  /* -(1000 + cudaError_t) */

typedef void* ner_stream_t; /* cudaStream_t */

const char* ner_strerror(int status);
/* Library/ABI version; bumps when a signature changes. */
int ner_abi_version(void);
/* Build provenance: "src=<hash of the sources this library was compiled from> nvcc=<version> arch=sm_90a"; the hash is
 * chinesener_b200.build.source_hash() of the tree at compile time. */
const char* ner_build_info(void);

/* ------------------------------------------------------------------------ *
 * CRF  — replaces tf.contrib.crf as called from tools/layer.py
 * ------------------------------------------------------------------------ */

/* tools/layer.py:140-142  crf_decode -> tf.contrib.crf.crf_decode
 * Viterbi max-plus recursion + backtrace.  logits [B,L,K] f32, seq_len [B]
 * i32, trans [K,K] f32 (trans[i*K+j] = score of i->j).  tags_out [B,L] i32 is
 * zero beyond seq_len; best_score [B] f32 may be NULL.  Ties resolve to the
 * lowest tag index; fp32 association order is (s[i]+trans[i][j]) then
 * +logits, so the tag indices are bit-exact with the reference.  K <= 32. */
int ner_crf_viterbi(const float* logits, const int32_t* seq_len, const float* trans,
                    int32_t* tags_out, float* best_score, int B, int L, int K,
                    ner_stream_t stream);

/* Which kernel ner_crf_viterbi runs for a call of this shape.  The choice is a pure function of the arguments below
 * (csrc/crf_viterbi.cu lists the kernels and their limits); nothing else, in particular no environment variable,
 * changes it.  logits_aligned = the logits pointer is 16-byte aligned; num_sms = multiprocessors of the device.  No
 * CUDA call is made, so it can be asked on a machine without a GPU.  NER_VIT_NONE: ner_crf_viterbi returns
 * NER_ERR_UNSUPPORTED (L too long for every kernel, or K outside 1..32). */
enum {
  NER_VIT_SMALL = 0,       /* lane-per-tag kernel, B <= 4096 */
  NER_VIT_TMA = 1,         /* thread-per-sequence, logits by TMA, backpointers in shared memory */
  NER_VIT_PARKED = 2,      /* thread-per-sequence, low backpointer nibbles parked in tags_out */
  NER_VIT_ONCHIP_128 = 3,  /* thread-per-sequence, backpointers in shared memory, 128 sequences per CTA */
  NER_VIT_ONCHIP_32 = 4,   /* the same kernel with 32 sequences per CTA */
  NER_VIT_SMALL_ANY_B = 5, /* lane-per-tag kernel for an L no thread-per-sequence kernel holds, B > 4096 */
  NER_VIT_NONE = 6
};
int ner_crf_viterbi_plan(int B, int L, int K, int logits_aligned, int num_sms);

/* tools/layer.py:122-127  crf_layer -> tf.contrib.crf.crf_log_likelihood
 * ll[b] = gold-path score - log-partition (forward-alpha recursion).
 * tags [B,L] i32.  alpha_ws: NULL, or [B,L,K] f32 that receives alpha_t for
 * the backward pass.  logz_out: NULL or [B] f32.
 * flags: bit0 = force the exact (per-column max) logsumexp path. */
int ner_crf_loglik_fwd(const float* logits, const int32_t* tags, const int32_t* seq_len,
                       const float* trans, float* ll, float* logz_out, float* alpha_ws,
                       int B, int L, int K, int flags, ner_stream_t stream);

/* Gradient of the log-likelihood (the reference gets it from tf.gradients,
 * tools/train_utils.py:314): for g_b = (d_ll ? d_ll[b] : 1) * scale,
 *   d_logits[b,t,j] = g_b * (1[y_t=j] - P(y_t=j|x))            (0 beyond seq_len)
 *   d_trans[i,j]   += sum_b g_b * (count_b(i->j) - sum_t P(y_{t-1}=i,y_t=j|x))
 * alpha_ws / logz come from ner_crf_loglik_fwd.  d_logits [B,L,K] is fully
 * written; d_trans [K,K] is ACCUMULATED into (caller zeroes it).  For the
 * reference loss mean(-ll) (model/bert_bilstm_crf.py:32) pass d_ll = NULL,
 * scale = -1/B. */
int ner_crf_loglik_bwd(const float* logits, const int32_t* tags, const int32_t* seq_len,
                       const float* trans, const float* alpha_ws, const float* logz,
                       const float* d_ll, float scale, float* d_logits, float* d_trans, int B,
                       int L, int K, ner_stream_t stream);

/* Partial-annotation CRF (Tsuboi et al., COLING 2008) in place of tools/layer.py:122-127's crf_log_likelihood when
 * the gold path is only known as a set of allowed tags per position.  label_mask [B,L] i32: bit j of label_mask[b,t]
 * allows tag j at t (bits >= K ignored, t >= seq_len ignored).
 *   ll[b] = logZ_A - logZ,  logZ_A = log-sum over the paths inside the allowed sets of exp(score)
 * A one-hot mask gives ner_crf_loglik_fwd's ll; a row whose every position allows all K tags gives exactly 0.0; an
 * empty set at some t < seq_len gives -inf; seq_len <= 0 gives 0.
 * logz: NULL or [B,2] f32 (logZ_A, logZ).  alpha_ws: NULL or [2,B,L,K] f32 (alpha_A, alpha) for the backward.
 * flags: bit0 = force the exact (per-column max) logsumexp path. */
int ner_crf_partial_loglik_fwd(const float* logits, const int32_t* label_mask, const int32_t* seq_len,
                               const float* trans, float* ll, float* logz, float* alpha_ws, int B, int L, int K,
                               int flags, ner_stream_t stream);

/* Gradient of ner_crf_partial_loglik_fwd's ll, for g_b = (d_ll ? d_ll[b] : 1) * scale:
 *   d_logits[b,t,j] = g_b * (P_A(y_t=j) - P(y_t=j))                  (0 beyond seq_len, 0 for a row with ll = -inf)
 *   d_trans[i,j]   += sum_b g_b * sum_t (P_A(y_{t-1}=i,y_t=j) - P(y_{t-1}=i,y_t=j))
 * alpha_ws [2,B,L,K] and logz [B,2] come from ner_crf_partial_loglik_fwd.  d_logits is fully written, d_trans is
 * accumulated into, as for ner_crf_loglik_bwd. */
int ner_crf_partial_loglik_bwd(const float* logits, const int32_t* label_mask, const int32_t* seq_len,
                               const float* trans, const float* alpha_ws, const float* logz, const float* d_ll,
                               float scale, float* d_logits, float* d_trans, int B, int L, int K, ner_stream_t stream);

/* CRF-to-CRF knowledge distillation, forward half (csrc/crf_distill.cu).  A teacher CRF (t_logits [B,L,K],
 * t_trans [K,K]) and a student CRF (s_logits, s_trans) over the same K tags define, at temperature tau = 1/inv_temp,
 * the path distributions p^tau(y) ~ exp(score(y) / tau).  One pass runs both forward recursions on the potentials
 * scaled by inv_temp as they are read, and writes:
 *   logz [B,2] f32: (logZ_T, logZ_S) of p^tau, 0 for seq_len <= 0;  alpha_ws [2,B,L,K] f32: (alpha_T, alpha_S).
 * Both are required and feed ner_crf_distill_bwd.  seq_len > L counts as L.  flags: bit0 = force the exact
 * (per-column max) logsumexp path; without it the scaled-probability step runs when both scaled transition
 * matrices span < 30 nats and are finite.  NER_ERR_INVALID_ARG for B < 0, L < 1, K < 1, inv_temp not a positive
 * finite number, or a null pointer (B > 0); NER_ERR_UNSUPPORTED for K > 32 or L > 4095.  B = 0 is a no-op. */
int ner_crf_distill_fwd(const float* t_logits, const float* t_trans, const float* s_logits, const float* s_trans,
                        const int32_t* seq_len, float inv_temp, float* logz, float* alpha_ws, int B, int L, int K,
                        int flags, ner_stream_t stream);

/* CRF-to-CRF knowledge distillation, backward half: both backward recursions in one reverse pass.  With mu / xi the
 * unary / pairwise marginals of p^tau and g_b = (d_kl ? d_kl[b] : 1) * scale:
 *   kl[b] = sum_t mu_T[t]·(x_T - x_S)[t] / tau + sum_{t>=1} xi_T[t]·(T_T - T_S) / tau - logZ_T + logZ_S   (KL(T||S))
 *   d_s_logits[b,t,j] = g_b * (mu_S[t][j] - mu_T[t][j]) / tau                       (0 beyond seq_len)
 *   d_s_trans[i,j]   += sum_b g_b * sum_{t>=1} (xi_S[t][i][j] - xi_T[t][i][j]) / tau
 * A term whose teacher marginal is 0 adds 0 to kl (a teacher transition of -inf).  seq_len <= 0: kl = 0, no gradient.
 * A teacher equal to the student gives kl = 0.0 and zero gradients exactly.  alpha_ws / logz from ner_crf_distill_fwd
 * with the same inputs; kl [B], d_s_logits [B,L,K] (fully written) and d_s_trans (accumulated into, as for
 * ner_crf_loglik_bwd) are required, d_kl is optional.  flags and error codes as ner_crf_distill_fwd. */
int ner_crf_distill_bwd(const float* t_logits, const float* t_trans, const float* s_logits, const float* s_trans,
                        const int32_t* seq_len, float inv_temp, const float* alpha_ws, const float* logz,
                        const float* d_kl, float scale, float* kl, float* d_s_logits, float* d_s_trans, int B, int L,
                        int K, int flags, ner_stream_t stream);

/* N-best extension of tools/layer.py:140-142's tf.contrib.crf.crf_decode: the N highest-scoring tag paths of every
 * sequence, best first (list Viterbi, csrc/crf_nbest.cu).  Row b decodes n = min(max(seq_len[b], 1), L) positions, as
 * ner_crf_viterbi does.  A path's score is the fp32 left-to-right sum s_0 = x[0][y_0],
 * s_t = (s_{t-1} + trans[y_{t-1}][y_t]) + x[t][y_t].  Ties: at each step the candidates (predecessor i, its rank r) are
 * ordered by s + trans descending, then lower i, then lower r; the final lists by score, then lower last tag, then
 * lower rank.  So rank 0 is ner_crf_viterbi's path and best_score bit for bit, and the N scores are the N largest
 * path scores.
 *   tags_out [B,N,L] i32: rank r of row b at tags_out[(b*N + r)*L ...], zero past n and in empty ranks;
 *   scores_out [B,N] f32: -inf in empty ranks;  count_out [B] i32 or NULL: min(N, K^n), the ranks filled.
 * workspace: backpointers, at least ner_crf_viterbi_nbest_workspace_bytes(B, L, K, N) = B*L*K*N*2 bytes (0 for B = 0).
 * Returns NER_ERR_UNSUPPORTED outside 1 <= K <= 32, 1 <= N <= 16; NER_ERR_INVALID_ARG for B < 0, L < 1 or a null
 * logits / seq_len / trans / tags_out / scores_out; NER_ERR_WORKSPACE for a missing or short workspace; B = 0 is a
 * no-op.  All checked before any CUDA call. */
size_t ner_crf_viterbi_nbest_workspace_bytes(int B, int L, int K, int N);
int ner_crf_viterbi_nbest(const float* logits, const int32_t* seq_len, const float* trans, int N, int32_t* tags_out,
                          float* scores_out, int32_t* count_out, void* workspace, size_t workspace_bytes, int B, int L,
                          int K, ner_stream_t stream);

/* Wide tag sets (csrc/crf_wide.cu): ner_crf_viterbi, ner_crf_loglik_fwd and ner_crf_loglik_bwd for
 * 1 <= K <= NER_MAX_TAGS_WIDE, with the same arguments, row rules (seq_len <= 0 decodes one position, seq_len > L
 * counts as L), alpha workspace, flags, d_ll / scale and d_trans accumulation.  Viterbi's tags and best_score are
 * bit-exact with ner_crf_viterbi where both run.  Viterbi also takes a backpointer workspace of at least
 * ner_crf_wide_viterbi_workspace_bytes(B, L, K) = B*L*K bytes (0 for B = 0).  NER_ERR_INVALID_ARG for B < 0, L < 1 or
 * a required null pointer (B > 0); NER_ERR_UNSUPPORTED for K outside 1..NER_MAX_TAGS_WIDE; NER_ERR_WORKSPACE for a
 * missing or short workspace; B = 0 is a no-op.  All checked before any CUDA call. */
#define NER_MAX_TAGS_WIDE 128
size_t ner_crf_wide_viterbi_workspace_bytes(int B, int L, int K);
int ner_crf_wide_viterbi(const float* logits, const int32_t* seq_len, const float* trans, int32_t* tags_out,
                         float* best_score, void* workspace, size_t workspace_bytes, int B, int L, int K,
                         ner_stream_t stream);
int ner_crf_wide_loglik_fwd(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
                            float* ll, float* logz_out, float* alpha_ws, int B, int L, int K, int flags,
                            ner_stream_t stream);
int ner_crf_wide_loglik_bwd(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
                            const float* alpha_ws, const float* logz, const float* d_ll, float scale, float* d_logits,
                            float* d_trans, int B, int L, int K, ner_stream_t stream);

/* Which kernel configuration the three wide entry points run for a call of this shape: W = 64 threads (K <= 64) or
 * 128, one CTA per G = 1 or 4 sequences (G = 4 from B >= 8 * num_sms).  A pure function of its arguments; no CUDA
 * call, no environment.  NER_CRF_WIDE_NONE for B < 1, L < 1, num_sms < 1 or K outside 1..NER_MAX_TAGS_WIDE. */
enum {
  NER_CRF_WIDE_64_G1 = 0,
  NER_CRF_WIDE_64_G4 = 1,
  NER_CRF_WIDE_128_G1 = 2,
  NER_CRF_WIDE_128_G4 = 3,
  NER_CRF_WIDE_NONE = 4
};
int ner_crf_wide_plan(int B, int L, int K, int num_sms);


/* ------------------------------------------------------------------------ *
 * Dense layers on wgmma tensor cores — replaces tf.layers.dense /
 * modeling.dense_layer inside BertModel (tools/layer.py:68-77), the logits
 * projection's big-M cousins and the LSTM input projection (tools/layer.py:35)
 * ------------------------------------------------------------------------ */
#define NER_EPI_F32 0            /* out f32  = acc + bias                    */
#define NER_EPI_BF16 1           /* out bf16 = acc + bias                    */
#define NER_EPI_GELU_TANH_BF16 2 /* out bf16 = gelu_tanh(acc + bias)         */
#define NER_EPI_GELU_ERF_BF16 3  /* out bf16 = gelu_erf(acc + bias)          */
#define NER_EPI_RELU_BF16 4      /* out bf16 = relu(acc + bias)              */
#define NER_EPI_RES_F32 5        /* out f32  = acc + bias + residual (f32)   */
#define NER_EPI_RES_RELU_F32 6   /* out f32  = relu(acc + bias + residual)   */
#define NER_EPI_DIAG_DISCARD 99  /* diagnostic only: accumulate, store nothing */

/* tile_n selectors of ner_gemm_bf16: 64/128/192/256 = one CTA per 128 x tile_n tile
 * (one CTA), whole tiles round-robin over the SMs; the 2CTA values = a cluster of two CTAs per 256 x N
 * tile (B tile TMA-multicast to both); the SK values = 128 x tile_n tiles with stream-K scheduling (every SM gets
 * the same number of k-blocks; split tiles are summed through an internal fp32 scratch). */
#define NER_TILE_2CTA_128 1128
#define NER_TILE_2CTA_256 1256
#define NER_TILE_SK_128 2128
#define NER_TILE_SK_256 2256
/* tile_n = 0 fits whole waves on the SMs (best latency of ONE GEMM).  NER_TILE_AUTO_THROUGHPUT takes the
 * tile with the best FLOP rate (128 x 256 when N % 256 == 0): the choice when several streams keep the
 * SMs busy, so a partial last wave is not idle time. */
#define NER_TILE_AUTO_THROUGHPUT 3000

/* out[M,N] = epilogue(A[M,K] · Wt[N,K]^T + bias[N]).  A and Wt are bf16,
 * K contiguous (Wt is the TF kernel [K,N] transposed once by
 * ner_pack_weight_bf16).  bias may be NULL.  K % 8 == 0, N % 32 == 0.
 * A, Wt, out 16-byte aligned; bias, residual 8-byte aligned (NER_ERR_INVALID_ARG otherwise).
 * tile_n: 0 = auto, or one of the selectors above. */
int ner_gemm_bf16(const void* A, const void* Wt, const float* bias, const float* residual,
                  void* out, int M, int N, int K, int epilogue, int tile_n,
                  ner_stream_t stream);

/* FP8 (OCP e4m3 "fn", max 448) dense layer with block scales, the inference-only FP8 encoder's QKV / FFN GEMMs:
 *   out[M,N] = epi( w_scale[n] · Σ_j a_scale[m,j] · (Σ_{k in [128j, 128j+128)} A[m,k] · Wt[n,k]) + bias[n] )
 * A e4m3 [M,K] row-major with f32 a_scale [M, K/128]; Wt e4m3 [N,K] (K contiguous, from ner_quantize_weight_e4m3) with
 * f32 w_scale [N].  Each 128-wide k-block is accumulated by wgmma and promoted into an fp32 accumulator.
 * epilogue: NER_EPI_BF16 (out bf16 [M,N] = acc + bias), or NER_EPI_GELU_TANH_E4M3 / NER_EPI_GELU_ERF_E4M3: out e4m3 [M,N]
 * = GELU(acc + bias) quantised per 1 x 128 block, with the block scales in out_scale [M, N/128] (scale = amax / 448, or 1
 * for an all-zero block; round to nearest even, saturating).  bias may be NULL.  K % 128 == 0 and N % 128 == 0, else
 * NER_ERR_UNSUPPORTED.  A, Wt, out 16-byte aligned; w_scale, bias 8-byte aligned. */
#define NER_EPI_GELU_TANH_E4M3 7 /* out e4m3 + block scales = gelu_tanh(acc + bias) (ner_gemm_e4m3 only) */
#define NER_EPI_GELU_ERF_E4M3 8  /* out e4m3 + block scales = gelu_erf(acc + bias)  (ner_gemm_e4m3 only) */
int ner_gemm_e4m3(const void* A, const float* a_scale, const void* Wt, const float* w_scale, const float* bias,
                  void* out, float* out_scale, int M, int N, int K, int epilogue, ner_stream_t stream);

/* TF dense kernel w_kn [K,N] f32 -> e4m3 [N,K] (K contiguous) with one scale per output channel:
 * w_scale[n] = max_k |W[k,n]| / 448 (1 for an all-zero column), wt[n,k] = e4m3(W[k,n] / w_scale[n]). */
int ner_quantize_weight_e4m3(const float* w_kn, void* wt_nk_e4m3, float* w_scale, int K, int N, ner_stream_t stream);

/* TF dense kernel [K,N] f32 -> bf16 [N,K] (K contiguous), the B-operand layout of
 * ner_gemm_bf16.  Done once per weight (or per optimizer step). */
int ner_pack_weight_bf16(const float* w_kn, void* wt_nk_bf16, int K, int N, ner_stream_t stream);
/* The same for a whole group of kernels in one launch, writing BOTH bf16 layouts a TRAIN step needs from one read of the fp32
 * weights: entry e = TF-layout f32 kernel src [K, N]; dst_kn_bf16 (nullable) receives the cast in place layout with row stride
 * ld_kn (the K-major operand of the data-gradient GEMMs; a column block of a fused matrix via the pointer offset), dst_nk_bf16
 * (nullable) the transposed [N, K] pack with row stride ld_nk (the operand of the forward GEMMs).  entries_device [count] and
 * tile_start_device [count + 1] (prefix sums of ceil(K/64) * ceil(N/64)) are DEVICE arrays; total_tiles = tile_start[count]. */
typedef struct {
  const float* src;
  int K;
  int N;
  void* dst_nk_bf16;
  int ld_nk;
  void* dst_kn_bf16;
  int ld_kn;
} ner_pack_entry;
int ner_pack_weights_group_bf16(const ner_pack_entry* entries_device, const int32_t* tile_start_device, int count,
                                int total_tiles, ner_stream_t stream);
/* Elementwise f32 -> bf16 (round to nearest even). */
int ner_cast_bf16(const float* src, void* dst_bf16, size_t n, ner_stream_t stream);

/* tf.layers.dense(units=label_size) — model/bert_bilstm_crf.py:26, model/bert_crf.py:20.
 * out[M,N] f32 = x[M,F] · W[F,N] + bias[N], N <= 32; x is f32 (x_is_bf16=0) or bf16;
 * W is the TF kernel layout [F,N] f32.  row_map: NULL, or [M] i32 — input row r is written to
 * output row row_map[r] (scatter of packed token rows back to the padded [B*L] layout). */
int ner_dense_small_n(const void* x, int x_is_bf16, const float* W, const float* bias, float* out,
                      int M, int F, int N, const int32_t* row_map, ner_stream_t stream);

/* tf.nn.embedding_lookup (model/bilstm_crf.py:24): out[tok, 0:E] = table[ids[tok]], row
 * stride ld_out >= E. */
int ner_embedding_lookup(const float* table, const int32_t* ids, float* out, int n_tok, int E,
                         int V, int ld_out, ner_stream_t stream);
/* f32 [M,D] (row stride ld_src) -> bf16 [M,Dp] zero-padded to the GEMM's K % 8 == 0. */
int ner_cast_pad_bf16(const float* src, void* dst_bf16, int M, int D, int Dp, int ld_src,
                      ner_stream_t stream);

/* Sequence packing plan (removes padding rows from the token-major activations; padded
 * positions never reach loss or pred_ids because the CRF ignores t >= seq_len).  mask [B,L] i32
 * must be a prefix mask (1 for t < len_b), as data/base_preprocess.py:166-174 builds it.
 * cu_seqlens [B+1]: exclusive prefix sum of the lengths; tok_src [B*L]: tok_src[cu[b]+t] = b*L+t. */
int ner_seq_pack_plan(const int32_t* mask, int32_t* cu_seqlens, int32_t* tok_src, int B, int L,
                      ner_stream_t stream);

/* f32 [M,D] (row stride ld_src) -> hi = bf16(x), lo = bf16(x - hi), both [M,Dp] zero-padded.
 * Operands of the fp32-accurate dense mode: out = A_hi·W_hi + A_hi·W_lo + A_lo·W_hi, three
 * ner_gemm_bf16 launches chained through the f32 residual epilogue (error ~2^-17 relative). */
int ner_split_bf16(const float* src, void* hi_bf16, void* lo_bf16, int M, int D, int Dp,
                   int ld_src, ner_stream_t stream);

/* fp32 self-attention for small heads with the optional TENER relative-position term
 * (tools/transformer/tener.py:12-119): scores[q,k] = (Q_q+u_h)·K_k [+ (Q_q+v_h)·R_{k-q+L}],
 * times `scale`; keys k >= seq_len[b] are masked; softmax; ·V.  Q/K/V are row-major
 * [B*L, ld*] f32 with head h at columns [h*head_dim, (h+1)*head_dim).  u/v [heads, head_dim]
 * or NULL; rel_table [2L, head_dim] (positions -L..L-1) or NULL.  Writes out_f32 and/or a
 * (hi, lo) bf16 pair, all [B*L, heads*head_dim]; rows q >= seq_len[b] are zero.
 * head_dim in {20, 32, 40, 64}, L <= 512. */
int ner_attention_f32(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                      const float* bias_u, const float* bias_v, const float* rel_table,
                      const int32_t* seq_len, float scale, float* out_f32, void* out_hi_bf16,
                      void* out_lo_bf16, int B, int L, int num_heads, int head_dim,
                      ner_stream_t stream);

/* ------------------------------------------------------------------------ *
 * BERT encoder pieces — bert_base.bert.modeling.BertModel as driven from
 * tools/layer.py:63-81 (pretrain_bert_embedding)
 * ------------------------------------------------------------------------ */

/* embedding_lookup + embedding_postprocessor: LN(word[ids] + type[seg] + pos[0:L]).
 * Tables f32: word [vocab,H], type [n_type,H], pos [max_pos,H]; ids/seg [B,L] i32
 * (seg may be NULL = all zero).  Writes f32 and/or bf16 [B*L,H] (either may be NULL).
 * Packed mode: tok_src [n_packed] (from ner_seq_pack_plan) selects the padded index of every
 * packed row; output has n_packed rows.  tok_src = NULL: padded mode, B*L rows. */
int ner_bert_embed_ln(const float* word_emb, const float* type_emb, const float* pos_emb,
                      const float* gamma, const float* beta, const int32_t* ids,
                      const int32_t* seg, float* out_f32, void* out_bf16, int B, int L, int H,
                      int vocab, int n_type, int max_pos, float eps, const int32_t* tok_src,
                      int n_packed, ner_stream_t stream);

/* LayerNorm over the last axis of (y + optional f32 residual) [M,H] -> f32 and/or bf16.
 * y is f32 (y_is_bf16 = 0) or bf16 (the dense layer's bf16 epilogue output).
 * modeling.layer_norm (eps 1e-12) and tools/transformer/modules.py:40-65 (eps = FLT_EPSILON). */
int ner_layernorm(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                  const float* beta, float* out_f32, void* out_bf16, int M, int H, float eps,
                  ner_stream_t stream);

/* ner_bert_embed_ln / ner_layernorm that also write the normalised row as e4m3 [M,H] with 1 x 128 block scales
 * out_scale [M, H/128] (the A operand of ner_gemm_e4m3), quantised from the same fp32 values out_f32 receives.
 * out_e4m3 and out_scale are required; out_f32 / out_bf16 may be NULL.  H % 128 == 0, else NER_ERR_UNSUPPORTED. */
int ner_bert_embed_ln_e4m3(const float* word_emb, const float* type_emb, const float* pos_emb,
                           const float* gamma, const float* beta, const int32_t* ids,
                           const int32_t* seg, float* out_f32, void* out_bf16, void* out_e4m3, float* out_scale,
                           int B, int L, int H, int vocab, int n_type, int max_pos, float eps,
                           const int32_t* tok_src, int n_packed, ner_stream_t stream);
int ner_layernorm_e4m3(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                       const float* beta, float* out_f32, void* out_bf16, void* out_e4m3, float* out_scale, int M,
                       int H, float eps, ner_stream_t stream);

/* ner_layernorm with BertModel's hidden dropout fused in front of the residual add:
 * out = LN(dropout(y) + residual), mask = the counter-based decisions of ner_dropout (element = row*H + col).
 * keep_prob = 1: identical to ner_layernorm. */
int ner_layernorm_dropout(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                          const float* beta, float* out_f32, void* out_bf16, int M, int H, float eps,
                          float keep_prob, uint64_t seed, ner_stream_t stream);

/* attention_layer core: ctx = softmax(Q K^T * scale + (1-mask)*mask_add) V per head.
 * qkv bf16 [B*L, 3*num_heads*head_dim] (Q | K | V blocks, heads contiguous inside each),
 * mask [B,L] i32 (1 = keep), ctx bf16 [B*L, num_heads*head_dim].  head_dim must be 64.
 * BERT: scale = 1/sqrt(64), mask_add = -10000.  Packed mode: cu_seqlens [B+1] non-NULL — sequence b
 * occupies rows [cu[b], cu[b+1]) of qkv/ctx, every key is valid, mask is ignored.
 * keep_prob < 1: attention_probs dropout of BertModel in training (probabilities scaled by
 * keep(seed; b, head, q, k) / keep_prob after the softmax); keep_prob = 1: inference.
 * n_rows: rows of qkv / ctx — the packed token count in packed mode (0 = unknown), B*L or 0 in padded mode.
 * keep_prob = 1 with known n_rows and L <= 256 runs on wgmma (S = Q K^T and O = P V accumulate in registers, Q/K/V
 * tiles arrive by TMA, V is consumed as an MN-major operand); otherwise a warp-level mma.sync kernel (ABI version 2). */
int ner_bert_attention(const void* qkv_bf16, const int32_t* mask, void* ctx_bf16, int B, int L,
                       int num_heads, int head_dim, float scale, float mask_add,
                       const int32_t* cu_seqlens, int n_rows, float keep_prob, uint64_t seed,
                       ner_stream_t stream);

/* Backward of ner_attention_f32 (TRAIN mode of tools/transformer/tener.py:12-119).  d_out f32 [B*L, ld_dout]
 * = dL/d out.  Writes dQ (all rows; zero for t >= seq_len) and ACCUMULATES into dK, dV (f32, layouts of K / V),
 * d_bias_u / d_bias_v [num_heads, head_dim] (nullable) — zero them first.  Scores are recomputed. */
int ner_attention_f32_bwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                          const float* bias_u, const float* bias_v, const float* rel_table,
                          const int32_t* seq_len, float scale, const float* d_out, int ld_dout,
                          float* dQ, int ld_dq, float* dK, int ld_dk, float* dV, int ld_dv,
                          float* d_bias_u, float* d_bias_v, int B, int L, int num_heads, int head_dim,
                          ner_stream_t stream);

/* Whole BertModel forward in one call (what tools/layer.py:68-77 gets from
 * modeling.BertModel(...).get_sequence_output()).  `layers` is a HOST array of per-layer
 * device pointers: dense kernels packed by ner_pack_weight_bf16 ([N,K] bf16; wqkv = the
 * query|key|value kernels concatenated along N), biases / LayerNorm parameters f32.
 * Padded mode: cu_seqlens = tok_src = NULL, outputs have B*L rows.  Packed mode: both from
 * ner_seq_pack_plan, n_packed = total tokens, outputs have n_packed rows.
 * out_f32 / out_bf16 [rows,H] receive sequence_output; workspace from the sizing call. */
typedef struct {
  int hidden_size, num_heads, intermediate_size, num_layers;
  int vocab_size, type_vocab_size, max_position;
  float ln_eps;   /* 1e-12 */
  int gelu_erf;   /* 0: tanh approximation (google-research/bert modeling.gelu), 1: erf */
  int gemm_tile;  /* tile_n passed to every ner_gemm_bf16 of the composite calls: 0 or NER_TILE_AUTO_THROUGHPUT */
} ner_bert_config;

typedef struct {
  const void* wqkv;  const float* bqkv;        /* [3H,H] bf16, [3H] */
  const void* wo;    const float* bo;          /* attention/output/dense */
  const float* ln1_gamma; const float* ln1_beta;
  const void* wi;    const float* bi;          /* intermediate/dense [I,H] bf16 */
  const void* wd;    const float* bd;          /* output/dense [H,I] bf16 */
  const float* ln2_gamma; const float* ln2_beta;
} ner_bert_layer_weights;

size_t ner_bert_encoder_workspace_bytes(const ner_bert_config* cfg, int rows);
int ner_bert_encoder_fwd(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                         const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                         const ner_bert_layer_weights* layers, const int32_t* ids,
                         const int32_t* mask, const int32_t* seg, int B, int L,
                         const int32_t* cu_seqlens, const int32_t* tok_src, int n_packed,
                         float* out_f32, void* out_bf16, void* workspace, size_t workspace_bytes,
                         ner_stream_t stream);

/* The same forward with FP8 dense layers (inference only): QKV, FFN1 and FFN2 run on ner_gemm_e4m3, their A operands
 * written by the LayerNorms (ner_bert_embed_ln_e4m3 / ner_layernorm_e4m3) and by FFN1's GELU -> e4m3 epilogue.  The
 * out-projection, attention, the f32 residual stream and LayerNorm arithmetic are those of ner_bert_encoder_fwd.
 * Same modes and outputs (the last LayerNorm writes f32 + bf16).  hidden_size and intermediate_size must be multiples of
 * 128, else NER_ERR_UNSUPPORTED. */
typedef struct {
  const void* wqkv;  const float* sqkv;  const float* bqkv;   /* [3H,H] e4m3, [3H] scales, [3H] bias */
  const void* wo;    const float* bo;                         /* attention/output/dense, [H,H] bf16 */
  const float* ln1_gamma; const float* ln1_beta;
  const void* wi;    const float* si;    const float* bi;     /* intermediate/dense [I,H] e4m3, [I], [I] */
  const void* wd;    const float* sd;    const float* bd;     /* output/dense [H,I] e4m3, [H], [H] */
  const float* ln2_gamma; const float* ln2_beta;
} ner_bert_layer_weights_fp8;

size_t ner_bert_encoder_fp8_workspace_bytes(const ner_bert_config* cfg, int rows);
int ner_bert_encoder_fwd_fp8(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                             const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                             const ner_bert_layer_weights_fp8* layers, const int32_t* ids,
                             const int32_t* mask, const int32_t* seg, int B, int L,
                             const int32_t* cu_seqlens, const int32_t* tok_src, int n_packed,
                             float* out_f32, void* out_bf16, void* workspace, size_t workspace_bytes,
                             ner_stream_t stream);

/* TRAIN-mode BertModel (is_training=True) as two calls: forward keeping every activation the backward
 * pass needs, and backward accumulating into the caller's gradient tensors (tf.gradients of
 * tools/train_utils.py:314 through the encoder).  Padded layout, rows = B*L.
 * Dropout: hidden_keep = 1 - hidden_dropout_prob (embedding output, attention-output dense, FFN-output
 * dense), attn_keep = 1 - attention_probs_dropout_prob; counter-based masks from `seed`, regenerated by
 * the backward call (same seed).  `saved` (ner_bert_train_saved_bytes) carries the activations from
 * forward to backward; `scratch` (ner_bert_train_scratch_bytes) is backward-only. */
typedef struct {
  /* TF-layout [K_in, N_out] bf16 casts of the dense kernels (ner_cast_bf16): B operands of the data-gradient GEMMs */
  const void* wqkv_kn; const void* wo_kn; const void* wi_kn; const void* wd_kn;
  /* gradient tensors, f32, accumulated into (TF shapes: kernels [in,out], biases [out]) */
  float* d_wq; float* d_wk; float* d_wv; float* d_bq; float* d_bk; float* d_bv;
  float* d_wo; float* d_bo; float* d_ln1_gamma; float* d_ln1_beta;
  float* d_wi; float* d_bi; float* d_wd; float* d_bd; float* d_ln2_gamma; float* d_ln2_beta;
} ner_bert_layer_grads;

size_t ner_bert_train_saved_bytes(const ner_bert_config* cfg, int rows);
size_t ner_bert_train_scratch_bytes(const ner_bert_config* cfg, int rows);
int ner_bert_encoder_train_fwd(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                               const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                               const ner_bert_layer_weights* layers, const int32_t* ids,
                               const int32_t* mask, const int32_t* seg, int B, int L,
                               float hidden_keep, float attn_keep, uint64_t seed, float* out_f32,
                               void* out_bf16, void* saved, size_t saved_bytes, ner_stream_t stream);
int ner_bert_encoder_train_bwd(const ner_bert_config* cfg, const float* emb_ln_gamma,
                               const ner_bert_layer_weights* layers, const ner_bert_layer_grads* grads,
                               float* d_word_emb, float* d_type_emb, float* d_pos_emb,
                               float* d_emb_ln_gamma, float* d_emb_ln_beta, const int32_t* ids,
                               const int32_t* mask, const int32_t* seg, int B, int L,
                               float hidden_keep, float attn_keep, uint64_t seed, const float* d_out,
                               const void* saved, size_t saved_bytes, void* scratch,
                               size_t scratch_bytes, ner_stream_t stream);
/* Sequence-packed TRAIN composites (cu_seqlens / tok_src / n_packed from ner_seq_pack_plan): the per-token kernels run on
 * the n_packed real tokens only — BertModel's work on [PAD] positions feeds nothing that bert_bilstm_crf / bert_crf read
 * (tools/layer.py:35 and :122,140 stop at seq_len) — and attention takes cu_seqlens.  ids / seg / out_f32 / out_bf16 /
 * d_out keep the padded [B*L, .] layout of the non-packed calls; [PAD] rows of the outputs are zero.  Same dropout seed
 * scheme (masks are indexed by packed element).  Workspaces: the two *_packed_* size functions below. */
size_t ner_bert_train_packed_saved_bytes(const ner_bert_config* cfg, int n_packed);
size_t ner_bert_train_packed_scratch_bytes(const ner_bert_config* cfg, int n_packed, int padded_rows);
int ner_bert_encoder_train_fwd_packed(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                                      const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                                      const ner_bert_layer_weights* layers, const int32_t* ids, const int32_t* seg,
                                      int B, int L, const int32_t* cu_seqlens, const int32_t* tok_src, int n_packed,
                                      float hidden_keep, float attn_keep, uint64_t seed, float* out_f32,
                                      void* out_bf16, void* saved, size_t saved_bytes, ner_stream_t stream);
int ner_bert_encoder_train_bwd_packed(const ner_bert_config* cfg, const float* emb_ln_gamma,
                                      const ner_bert_layer_weights* layers, const ner_bert_layer_grads* grads,
                                      float* d_word_emb, float* d_type_emb, float* d_pos_emb,
                                      float* d_emb_ln_gamma, float* d_emb_ln_beta, const int32_t* ids,
                                      const int32_t* seg, int B, int L, const int32_t* cu_seqlens,
                                      const int32_t* tok_src, int n_packed, float hidden_keep, float attn_keep,
                                      uint64_t seed, const float* d_out, const void* saved, size_t saved_bytes,
                                      void* scratch, size_t scratch_bytes, ner_stream_t stream);
/* Row moves between the padded and the packed layouts (row_bytes a multiple of 16):
 * gather: dst row r = src row idx[r];  scatter: dst row idx[r] = src row r (rows not named keep their content). */
int ner_gather_rows(const void* src, const int32_t* idx, void* dst, int n, int row_bytes, ner_stream_t stream);
int ner_scatter_rows(const void* src, const int32_t* idx, void* dst, int n, int row_bytes, ner_stream_t stream);
/* word[ids] + type[seg] + pos[0:L] without the LayerNorm -> f32 [B*L,H] (operand of the embedding
 * LayerNorm backward). */
int ner_bert_embed_sum(const float* word_emb, const float* type_emb, const float* pos_emb,
                       const int32_t* ids, const int32_t* seg, float* out, int B, int L, int H,
                       int vocab, int n_type, int max_pos, ner_stream_t stream);

/* The whole PREDICT step of model/bert_bilstm_crf.py:8-34 in one call (what a PREDICT session.run
 * of that plugin executes: BertModel -> bilstm -> dense(logits) -> crf_decode; the log-likelihood
 * is not fetched in PREDICT).  Same kernels, same order as the layer-by-layer entry points above.
 * lstm_wx_bf16 [8*lstm_hidden, H] = ner_pack_weight_bf16 of [kernel_fw[:H] | kernel_bw[:H]],
 * lstm_bias [8*lstm_hidden] = [bias_fw | bias_bw], lstm_wh_* = kernel[H:, :] f32,
 * lstm_activation as ner_bilstm_recurrence, logits_w [2*lstm_hidden, num_tags], trans [K,K].
 * n_packed = number of valid tokens (sum of mask), known on the host; pred_ids [B,L] i32. */
size_t ner_bert_bilstm_crf_predict_workspace_bytes(const ner_bert_config* cfg, int B, int L, int rows,
                                                   int lstm_hidden, int num_tags);
int ner_bert_bilstm_crf_predict(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                                const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                                const ner_bert_layer_weights* layers, const void* lstm_wx_bf16,
                                const float* lstm_bias, const float* lstm_wh_fw, const float* lstm_wh_bw,
                                int lstm_hidden, int lstm_activation, const float* logits_w,
                                const float* logits_b, const float* trans, int num_tags,
                                const int32_t* ids, const int32_t* mask, const int32_t* seg,
                                const int32_t* seq_len, int B, int L, int n_packed, int32_t* pred_ids,
                                void* workspace, size_t workspace_bytes, ner_stream_t stream);

/* ------------------------------------------------------------------------ *
 * BiLSTM — tools/layer.py:27-41 bilstm() -> bidirectional_dynamic_rnn(LSTMCell)
 * ------------------------------------------------------------------------ */

/* Sequential half of both directions.  xproj [B*L, 8H] f32 = x · [kernel_fw[:D] | kernel_bw[:D]]
 * + [bias_fw | bias_bw] (one ner_gemm_bf16 call, NER_EPI_F32); wh_fw / wh_bw = kernel[D:, :]
 * [H,4H] f32 with TF's gate order (i, j, f, o).  out [B,L,2H] f32 = concat(fw, bw), zero for
 * t >= seq_len.  activation: 0 tanh, 1 relu (params['rnn_activation']).  H % 4 == 0.
 * cu_seqlens: NULL (xproj row of (b,t) = b*L+t) or [B+1] (packed xproj: row = cu[b]+t).
 * gates_out [B*L, 8H] / cstate_out [B,L,2H]: both NULL (inference) or both given (training):
 * post-activation gates (sigmoid(i), act(j), sigmoid(f+forget_bias), sigmoid(o)) and cell states.
 * keep_prob < 1 (training, tools/layer.py:20-23 DropoutWrapper(output_keep_prob, state_keep_prob)):
 * independent counter-based masks (seed) on the emitted output and on the carried h; hstate_out
 * [B,L,2H] (nullable) receives the carried (state-dropped) h, the operand of dW_h. */
int ner_bilstm_recurrence(const float* xproj, const float* wh_fw, const float* wh_bw,
                          const int32_t* seq_len, float* out, int B, int L, int H,
                          int activation, float forget_bias, const int32_t* cu_seqlens,
                          float* gates_out, float* cstate_out, float* hstate_out, float keep_prob,
                          uint64_t seed, ner_stream_t stream);

/* Back-propagation through time of ner_bilstm_recurrence (padded layout).  d_out [B,L,2H] f32;
 * gates [B*L, 8H] / cstate [B,L,2H] saved by the forward call.  Writes d_xproj [B*L, 8H] f32 =
 * gradient w.r.t. the hoisted input projection (zeros for t >= seq_len).  The caller finishes
 * with plain GEMMs / reductions over it: dW_x = x^T d_xproj, d_bias = colsum(d_xproj),
 * dx = d_xproj W_x^T, dW_h = h_prev^T d_xproj (per direction). */
int ner_bilstm_recurrence_bwd(const float* d_out, const float* gates, const float* cstate,
                              const float* wh_fw, const float* wh_bw, const int32_t* seq_len,
                              float* d_xproj, int B, int L, int H, int activation, float keep_prob,
                              uint64_t seed, ner_stream_t stream);

/* ------------------------------------------------------------------------ *
 * BiGRU — tools/layer.py:10-41 bilstm(cell_type='gru') -> bidirectional_dynamic_rnn(GRUCell)
 * ------------------------------------------------------------------------ */

/* Sequential half of both directions of TF 1.14 GRUCell (r, u = sigmoid(split([x,h]·Wg + bg)); c = act([x, r⊙h]·Wc + bc);
 * h' = u⊙h + (1-u)⊙c).  xproj [rows, 6H] f32 = x · [Wg_fw[:D] | Wc_fw[:D] | Wg_bw[:D] | Wc_bw[:D]] + biases (one
 * ner_gemm_bf16 call) with row stride ld_xproj >= 6H (the GEMM needs N % 32 == 0: its weight pack is padded with zero
 * columns when H % 16 != 0); wh_fw / wh_bw [H,3H] f32 = [gates/kernel[D:] | candidate/kernel[D:]] (columns r, u, c).
 * out [B,L,2H] f32 = concat(fw, bw), zero for t >= seq_len.  activation: 0 tanh, 1 relu.  H % 4 == 0 and H small
 * enough for the recurrent slice to fit an 8-CTA cluster (every H <= 256), else NER_ERR_UNSUPPORTED.  cu_seqlens as
 * ner_bilstm_recurrence.  gates_out [B*L, 6H], hstate_out [B,L,2H], rh_out [B,L,2H]: all NULL (inference) or all given
 * (training): post-activation r, u, c, the carried (state-dropped) h and r ⊙ h_prev (the operand of dW_c^h).
 * keep_prob < 1: DropoutWrapper(output_keep_prob, state_keep_prob) with independent counter-based masks (seed) on the
 * output and on the carried state, the masks of ner_bilstm_recurrence. */
int ner_bigru_recurrence(const float* xproj, const float* wh_fw, const float* wh_bw, const int32_t* seq_len,
                         float* out, int B, int L, int H, int ld_xproj, int activation,
                         const int32_t* cu_seqlens, float* gates_out, float* hstate_out, float* rh_out, float keep_prob, uint64_t seed,
                         ner_stream_t stream);

/* Back-propagation through time of ner_bigru_recurrence (padded layout; TF GRUCell over tools/layer.py:10-41).
 * d_out [B,L,2H]; gates [B*L, 6H] and hstate [B,L,2H] saved by the forward call.  Writes d_xproj [B*L, 6H] f32
 * (columns da_r, da_u, da_c per direction; zeros for t >= seq_len).  The caller finishes with GEMMs / column sums over
 * it: dW_x = x^T d_xproj, d_bias = colsum(d_xproj), dx = d_xproj W_x^T, dW_g^h = h_prev^T da_g, dW_c^h = (r⊙h_prev)^T
 * da_c. */
int ner_bigru_recurrence_bwd(const float* d_out, const float* gates, const float* hstate, const float* wh_fw,
                             const float* wh_bw, const int32_t* seq_len, float* d_xproj, int B, int L, int H,
                             int activation, float keep_prob, uint64_t seed, ner_stream_t stream);

/* Which instantiation a recurrence call runs (csrc/rnn_plan.cu holds the rules).  The launchers of the six kernels
 * below (ner_bilstm_recurrence, _bwd, ner_bigru_recurrence, _bwd, ner_lattice_recurrence, _bwd) call it with the
 * device's SM count and launch what it returns, so the answer for a shape is the launch.  Out: *rows = batch rows per
 * cluster (the kernel's template R), *cluster = CTAs per cluster, *resident = 1 when the recurrent matrix is held in
 * registers (LSTM at H = 128) and 0 otherwise; each may be NULL.  Kw (words per lattice position) is read only for
 * the lattice kernels.  Returns NER_OK, or the status the launcher returns for that shape before any CUDA call
 * (NER_ERR_INVALID_ARG for B < 0, H < 1, num_sms < 1, Kw < 1 (lattice) or an unknown kernel; NER_ERR_UNSUPPORTED
 * for an H no cluster holds, H % 4 != 0 (LSTM forward, GRU) or Kw > 8), with the outputs set to 0.  A pure host
 * function: no CUDA call and no environment variable enters it. */
enum {
  NER_RNN_LSTM_FWD = 0,
  NER_RNN_LSTM_BWD = 1,
  NER_RNN_GRU_FWD = 2,
  NER_RNN_GRU_BWD = 3,
  NER_RNN_LATTICE_FWD = 4,
  NER_RNN_LATTICE_BWD = 5
};
int ner_rnn_plan(int kernel, int B, int H, int Kw, int num_sms, int* rows, int* cluster, int* resident);

/* ------------------------------------------------------------------------ *
 * SoftLexicon gather-and-pool — model/bilstm_crf_softlexicon.py:37-44
 * ------------------------------------------------------------------------ */

/* out[tok, g*E+e] = sum_s weights[tok, g*S+s] * table[ids[tok, g*S+s], e].
 * table [V,E] f32, ids/weights [n_tok, G*S], out [n_tok, G*E] with row stride ld_out
 * (>= G*E; lets the caller pool straight into a concat buffer).  G*S <= 64, E <= 128. */
int ner_softlexicon_pool_fwd(const float* table, const int32_t* ids, const float* weights,
                             float* out, int n_tok, int G, int S, int E, int V, int ld_out,
                             ner_stream_t stream);
/* d_table [V,E] += scatter of weights * d_out (caller zeroes / owns accumulation). */
int ner_softlexicon_pool_bwd(float* d_table, const int32_t* ids, const float* weights,
                             const float* d_out, int n_tok, int G, int S, int E, int V,
                             ner_stream_t stream);

/* ------------------------------------------------------------------------ *
 * Small-table word-enhance embeddings — model/bilstm_crf_softword.py, model/bilstm_crf_ex_softword.py
 * ------------------------------------------------------------------------ */

/* ExSoftword projection: out[t, 0:E] = sum_v weights[t, v] * table[v, :], summed over v ascending, zero weights skipped.
 * table [V,E] f32, weights [n_tok,V] f32, out row stride ld_out >= E (lets the caller write into a concat buffer).
 * V <= 8 and E <= 128, else NER_ERR_UNSUPPORTED.  Null pointers are NER_ERR_INVALID_ARG unless n_tok == 0. */
int ner_multihot_embed_fwd(const float* table, const float* weights, float* out, int n_tok, int V, int E,
                           int ld_out, ner_stream_t stream);
/* Gradient of a [V,E] table read by ner_embedding_lookup (ids) or ner_multihot_embed_fwd (weights):
 *   d_table[v, :] += sum_t c(t, v) * d_out[t, :],  c(t, v) = [clamp(ids[t], 0, V-1) == v]  or  weights[t, v].
 * Exactly one of ids [n_tok] i32 / weights [n_tok,V] f32 is given (both, or neither with n_tok > 0, is
 * NER_ERR_INVALID_ARG); ids outside [0, V) are clamped into it, as the SoftLexicon pool does.  d_out row stride
 * ld_dout >= E.  V <= 8 and E <= 128, else NER_ERR_UNSUPPORTED.  Deterministic, no float atomics: each CTA sums a fixed
 * token range into a [V,E] partial in `scratch` (>= ner_small_table_grad_scratch_floats(V, E) floats, 0 for an
 * unsupported V, E), and the partials are added in CTA order.  The grid depends only on n_tok and the SM count, so a
 * device gives a bit-identical gradient on every call. */
size_t ner_small_table_grad_scratch_floats(int V, int E);
int ner_small_table_grad(float* d_table, const int32_t* ids, const float* weights, const float* d_out, int n_tok,
                         int V, int E, int ld_dout, float* scratch, ner_stream_t stream);

/* ------------------------------------------------------------------------ *
 * Training-side kernels — gradients of the layers above and the two optimizer steps of
 * tools/train_utils.py:246-390
 * ------------------------------------------------------------------------ */

/* src f32 [M,N] (row stride ld_src) -> bf16 [N,Mp] zero-padded: K-major operand of a
 * weight-gradient GEMM dW[K,N] = X^T dY (the reduction runs over the M rows). */
int ner_transpose_cast_bf16(const float* src, void* dst_bf16, int M, int N, int Mp, int ld_src,
                            ner_stream_t stream);
/* out[n] += scale * sum_m x[m,n]  (bias gradients). */
int ner_colsum_add(const float* x, float* out, int M, int N, int ld, float scale,
                   ner_stream_t stream);
/* Gradient of ner_dense_small_n (f32 x): dW [F,N] += x^T dy, db [N] += colsum(dy) (db may be
 * NULL), dx [M,F] = dy W^T (dx may be NULL).  dW/db are accumulated into (caller zeroes). */
int ner_dense_small_n_bwd(const float* x, const float* W, const float* dy, float* dW, float* db,
                          float* dx, int M, int F, int N, ner_stream_t stream);
/* tf.layers.dropout: y[i] = keep(seed, i) ? x[i]/keep_prob : 0.  Counter-based: the same
 * (seed, i) reproduces the mask, so the backward pass is the same call on the gradient. */
int ner_dropout(const float* x, float* y, size_t n, float keep_prob, uint64_t seed,
                ner_stream_t stream);
/* Same on bf16 tensors (BertModel's hidden dropout on the bf16 dense outputs; y may alias x). */
int ner_dropout_bf16(const void* x_bf16, void* y_bf16, size_t n, float keep_prob, uint64_t seed,
                     ner_stream_t stream);
/* tf.nn.relu on f32 [n] (y may alias x). */
int ner_relu_f32(const float* x, float* y, size_t n, ner_stream_t stream);
/* tf.nn.relu gradient: dpre = dact where act > 0 else 0 (f32 [n]; dpre may alias dact). */
int ner_relu_bwd_f32(const float* act, const float* dact, float* dpre, size_t n, ner_stream_t stream);
/* tf.reduce_max(x[B,L,C], axis=1) -> y[B,C] (reference model/bert_bilstm_crf_adv.py:35, the task discriminator's pool). */
int ner_reduce_max_time(const float* x, float* y, int B, int L, int C, ner_stream_t stream);
/* Its TF gradient, accumulated: dx[b,t,c] += scale * dy[b,c] / ties wherever x[b,t,c] == y[b,c]
 * (scale = -shrink_gradient_reverse folds FlipGradientBuilder, tools/train_utils.py:47-63). */
int ner_reduce_max_time_bwd(const float* x, const float* y, const float* dy, float* dx, int B, int L, int C,
                            float scale, ner_stream_t stream);
/* tf.nn.sparse_softmax_cross_entropy_with_logits (model/bert_bilstm_crf_adv.py:46) on [B, N <= 32]:
 * loss[b]; dlogits (nullable) = scale * (softmax - onehot). */
int ner_softmax_xent(const float* logits, const int32_t* labels, float* loss, float* dlogits, int B, int N,
                     float scale, ner_stream_t stream);
/* model/bert_ce.py + tools/loss.py: cross_entropy_loss and tf.argmax(logits, -1) in one pass over logits [B,L,K] f32.
 * pred_ids [B,L] i32 (nullable): first argmax at EVERY t < L (not masked).  labels [B,L] i32 (nullable: no loss).
 * loss [1] f32 (nullable) = sum_{t<len_b} (lse - z[y]) / N,  N = sum_b clamp(len_b, 0, L), 0 when N = 0.
 * d_logits [B,L,K] f32 (nullable, fully written) = d_loss / N * (softmax - onehot) for t < len_b, 0 elsewhere.
 * Deterministic: per-CTA partials in scratch (>= ner_token_xent_scratch_floats()), summed in index order; no float
 * atomics.  N is computed on the device from seq_len (no host synchronisation).  K <= 32; labels in [0, K) for t < len_b.
 * seq_len and scratch are required with labels; loss / d_logits without labels is NER_ERR_INVALID_ARG.  B * L < 2^31. */
size_t ner_token_xent_scratch_floats(void);
int ner_token_xent(const float* logits, const int32_t* labels, const int32_t* seq_len, int32_t* pred_ids, float* loss,
                   float* d_logits, float d_loss, float* scratch, int B, int L, int K, ner_stream_t stream);
/* model/bert_dice.py + tools/loss.py: dice_loss and tf.argmax(logits, -1) in one pass over logits [B,L,K] f32, the same
 * pass as ner_token_xent with the self-adjusting Dice loss (Li et al., "Dice Loss for Data-imbalanced NLP Tasks", ACL 2020)
 * applied to every class of every token t < len_b.  With p = softmax(z), u_k = 1 - p_k, q_k = u_k^alpha * p_k (u^0 = 1):
 *   l = sum_k l_k,  l_y = (1 - q_y) / (q_y + 1 + gamma),  l_k = q_k / (q_k + gamma) for k != y
 *     (= 1 - (2 q_k [k=y] + gamma) / (q_k + [k=y] + gamma), the paper's form)
 * loss [1] f32 (nullable) = sum_{t<len_b} l / N,  N = sum_b clamp(len_b, 0, L), 0 when N = 0.
 * d_logits [B,L,K] f32 (nullable, fully written) = d_loss / N * d l / d z for t < len_b, 0 elsewhere, computed as
 *   c_k = d l_k / d q_k * p_k * u_k^alpha * (u_k - alpha p_k),  r_k = c_k / s_{-k},  d l / d z_j = c_j - e_j (sum_k r_k - r_j)
 * with e = exp(z - max z), s_{-k} = sum_{i != k} e_i and u_k = s_{-k} / sum e (never 1 - p_k, which is 0 in fp32 on a
 * confident row).  pred_ids (nullable) as ner_token_xent.  labels, seq_len and scratch (ner_token_xent_scratch_floats())
 * are required; alpha >= 0 and gamma > 0 finite, else NER_ERR_INVALID_ARG; otherwise the checks of ner_token_xent.
 * Deterministic like ner_token_xent.  The reference's tools/loss.py is not in this repository: the loss, its token-mean
 * reduction and the plugin's defaults alpha = gamma = 1 are a restatement of the paper, not pinned to the reference. */
int ner_token_dice(const float* logits, const int32_t* labels, const int32_t* seq_len, int32_t* pred_ids, float* loss,
                   float* d_logits, float d_loss, float alpha, float gamma, float* scratch, int B, int L, int K,
                   ner_stream_t stream);
/* ---- masked-LM pretraining (chinesener_b200/mlm.py; a restatement of google-research/bert's create_pretraining_data.py
 * and run_pretraining.py, not pinned to them) ---- */
#define NER_MLM_MAX_LEN 512       /* L of ner_mlm_mask */
#define NER_MLM_MAX_VOCAB 50000   /* V of both entry points */
/* Dynamic whole-word masking of token_ids [B,L] i32.  Row b: n = clamp(seq_len[b], 0, L); candidates are the positions
 * 1 .. n-2 ([CLS] at 0 and [SEP] at n-1 are never chosen).  A word is a maximal run of candidates starting at a position
 * with word_start[b,t] = 1 (or at position 1) followed by positions with word_start = 0; word_start [B,L] u8 NULL makes
 * every candidate its own word.  With h_k(b, t) = hash3(lo(seed) + k * 0x9E3779B9, hi(seed) ^ b, t) (common.cuh), word w
 * starting at s_w gets the key h_0(b, s_w); the words are walked in (key, s_w) order and a word is taken when
 * taken + |w| <= k_b, else skipped (k_b = pred_offsets[b+1] - pred_offsets[b], the row's budget, computed by the caller).
 * Every position t of a taken word is a prediction: with u = (h_1(b, t) >> 8) / 2^24, masked_ids[b,t] = mask_id for
 * u < 0.8, umulhi(h_2(b, t), V) (a uniform id in [0, V)) for 0.8 <= u < 0.9, else token_ids[b,t]; every other element
 * of masked_ids is token_ids.  positions / labels [M = pred_offsets[B]] i32: from pred_offsets[b] on, b*L + t and
 * token_ids[b,t] of row b's predictions in ascending t, then its unused slots (skipped words can leave fewer than k_b)
 * with b*L and -1.  B < 0, L < 1, V < 1, mask_id outside [0, V) or a null pointer (word_start aside) is
 * NER_ERR_INVALID_ARG; L > NER_MLM_MAX_LEN, V > NER_MLM_MAX_VOCAB or B*L >= 2^31 is NER_ERR_UNSUPPORTED; all before any
 * CUDA call.  B = 0 is a no-op.  One launch, no allocation, no atomics, bit-identical repeats. */
int ner_mlm_mask(const int32_t* token_ids, const int32_t* seq_len, const uint8_t* word_start, const int32_t* pred_offsets,
                 int B, int L, uint64_t seed, int V, int mask_id, int32_t* masked_ids, int32_t* positions, int32_t* labels,
                 ner_stream_t stream);
/* Masked-LM loss, gradient and argmax over logits [M, ld] f32 (columns 0 .. V-1 are the classes).  A row is counted when
 * 0 <= labels[r] < V; other labels, -1 included, add nothing to any output but pred.  count [1] = the counted rows;
 * loss [1] = sum over counted rows of (logsumexp(z) - z[y]) / count, 0 when count = 0; correct [1] = counted rows whose
 * first argmax equals the label; pred [M] (nullable) = the first argmax of every row.  d_logits [M, ld] bf16 (nullable,
 * fully written) = d_loss / count * (softmax(z) - onehot(y)) on counted rows in columns < V, exactly 0 elsewhere.
 * Deterministic: per-row losses in scratch (>= ner_vocab_xent_scratch_floats(M) floats) summed in index order; no float
 * atomics; the count is taken on the device.  M < 0, V < 1, ld < V, ld % 4 != 0, a logits pointer not 16-byte aligned, a
 * d_logits pointer not 8-byte aligned or a null logits / labels / loss / count / correct / scratch is NER_ERR_INVALID_ARG;
 * V > NER_MLM_MAX_VOCAB is NER_ERR_UNSUPPORTED; all before any CUDA call.  M = 0 is a no-op.  Three launches. */
size_t ner_vocab_xent_scratch_floats(int M);
int ner_vocab_xent(const float* logits, int ld, const int32_t* labels, int M, int V, float d_loss, float* loss,
                   int32_t* count, int32_t* correct, int32_t* pred, void* d_logits, float* scratch, ner_stream_t stream);
/* ---- training-data augmentation (chinesener_b200/augment.py; Dai & Adel, COLING 2020, and masked-LM replacement after
 * Kobayashi, NAACL 2018) ---- */
#define NER_AUGMENT_MAX_LEN 4095      /* L of ner_augment_rows */
#define NER_AUGMENT_MLM_BUDGET 20     /* masked-LM replacements per row */
/* Augments a BIO batch token_ids / label_ids / mask / segment_ids [B,L] i32, seq_len [B] i32 into the *_out arrays (not
 * in place).  h_k(b, t) = hash3(lo(seed) + k * 0x9E3779B9, hi(seed) ^ b, t); "drawn with p" means
 * (h >> 8) < (uint32)(p * 2^24); "pick from n" means umulhi(h, n).  Streams k: 0 row, 1 / 2 MR choice / draw, 3 / 4
 * LwTR choice / draw, 5 / 6 SiS choice / key, 7 MLM choice, 8 ner_vocab_sample's Gumbel draws.
 * tag_class [K] gives each tag id its class: 0 special (never touched), 1 O, 2 + 2x B of type x, 3 + 2x I of type x;
 * a label outside [0, K) is special.  type_tag [T, 2] = (B id, I id or -1) of type x.  Pools (CSR, offsets relative to
 * their arrays, a malformed range is an empty pool): mention_type_off [T+1] into the mention list, mention_tok_off
 * [n_mentions+1] into mention_tokens [n_mention_tokens]; tag_tok_off [K+1] into tag_tokens [n_tag_tokens].
 * Row b is augmented when h_0(b, 0) is drawn with p_row; any other row is copied unchanged (seq_len included).  For an
 * augmented row with n = clamp(seq_len[b], 0, L), in this order:
 *   MR   A mention is a B-x token and the run of I-x tokens after it (span::run_end).  Mentions left to right; with s the
 *        mention's start in the input row, the mention is chosen when h_1(b, s) is drawn with p_mr, and replaced by
 *        mention pick(h_2(b, s), count of type x) of type x's pool (tags B-x, I-x ...) when the row's running length
 *        minus the old plus the new mention's length stays <= L; otherwise it stays.  Other tokens are copied.
 *   LwTR Every non-special position t of the new row with h_3(b, t) drawn with p_lwtr takes the token
 *        pick(h_4(b, t), count) of its tag's pool (unchanged when that pool is empty).
 *   SiS  Segments of the new row: a mention, a maximal run of O, or any other single token (a stray I-x, a special tag).
 *        A segment starting at s with length >= 2 is chosen when h_5(b, s) is drawn with p_sis; its tokens are reordered
 *        by ascending (h_6(b, t), t) of their positions t.  Tags stay in place.
 *   MLM  (mlm_ids non-NULL) The first NER_AUGMENT_MLM_BUDGET O positions t, ascending, with h_7(b, t) drawn with p_mlm:
 *        mlm_ids holds mask_id there and the row elsewhere; mlm_positions [B, NER_AUGMENT_MLM_BUDGET] holds b*L + t of
 *        them in order, then -1 (all -1 in a row that is not augmented).
 * Outputs of an augmented row with new length n': token / label ids of the row, then pad_id / pad_tag; mask 1 below n'
 * and 0 from it; segment ids 0; seq_len_out = n'.  B < 0, L < 1, K < 1, T < 0, a probability outside [0, 1], a negative
 * pool size, p_mlm > 0 without mlm_ids, only one of mlm_ids / mlm_positions, mask_id < 0 with them, or a null pointer an
 * enabled operation reads is NER_ERR_INVALID_ARG; L > NER_AUGMENT_MAX_LEN, K > NER_MAX_TAGS_WIDE or B*L >= 2^31 is
 * NER_ERR_UNSUPPORTED; all before any CUDA call.  B = 0 is a no-op.  One launch with
 * ner_augment_rows_smem_bytes(L) bytes of dynamic shared memory, no allocation, bit-identical repeats. */
size_t ner_augment_rows_smem_bytes(int L);
int ner_augment_rows(const int32_t* token_ids, const int32_t* label_ids, const int32_t* seq_len, const int32_t* mask,
                     const int32_t* segment_ids, int B, int L, const int32_t* tag_class, int K, const int32_t* type_tag,
                     int T, const int32_t* mention_type_off, const int32_t* mention_tok_off, const int32_t* mention_tokens,
                     int n_mentions, int n_mention_tokens, const int32_t* tag_tok_off, const int32_t* tag_tokens,
                     int n_tag_tokens, float p_row, float p_mr, float p_lwtr, float p_sis, float p_mlm, uint64_t seed,
                     int pad_id, int pad_tag, int mask_id, int32_t* token_out, int32_t* label_out, int32_t* seq_len_out,
                     int32_t* mask_out, int32_t* segment_out, int32_t* mlm_ids, int32_t* mlm_positions,
                     ner_stream_t stream);
/* Gumbel-max sample of one id per slot r < M from softmax(logits[r, :V] / temperature) restricted to the ids j with
 * eligible[j] != 0 and j != token_ids[positions[r]]: argmax_j logits[r, j] / temperature - log(-log(u_j)), u_j =
 * ((h_8(positions[r], j) >> 9) + 0.5) / 2^23 in fp32 (ties to the lower id).  The id is written to
 * token_ids[positions[r]]; a slot with positions[r] outside [0, n_tokens) is skipped, and a row without an eligible id
 * leaves its token.  logits [M, ld] f32, 16-byte aligned, ld % 4 == 0.  M < 0, V < 1, ld < V, ld % 4 != 0,
 * n_tokens < 0, a temperature that is not a positive finite number, a misaligned logits or a null pointer is
 * NER_ERR_INVALID_ARG; V > NER_MLM_MAX_VOCAB is NER_ERR_UNSUPPORTED; all before any CUDA call.  M = 0 is a no-op. */
int ner_vocab_sample(const float* logits, int ld, int V, const uint8_t* eligible, const int32_t* positions, int M,
                     long long n_tokens, float temperature, uint64_t seed, int32_t* token_ids, ner_stream_t stream);
/* model/bert_mrc.py (MRC-style NER, one BERT query per entity type; a restatement, not pinned to the reference's mrc/):
 * expands the [B,L] BERT batch (token_ids, seq_len [B] counting [CLS] and [SEP]) into the B*T pairs p = b*T + t,
 *   pair row p = token_ids[b,0] ([CLS]), query_ids[t, 0:q_t], sep_id, token_ids[b, 1:len_b]
 * of n_p = q_t + 1 + len_b tokens (0 when len_b = 0), len_b = clamp(seq_len[b], 0, L), q_t = clamp(query_len[t], 0, Qmax).
 * query_ids [T,Qmax] i32 (may be NULL when Qmax = 0), query_len [T] i32, type_tag [T,2] i32 = tag ids of (B-X_t, I-X_t).
 * Writes pair_ids / pair_segment_ids / pair_mask [B*T, L2] i32 (segment 0 up to and including the query's [SEP], 1 after;
 * mask 1 for j < n_p; all three 0 from n_p on), pair_seq_len [B*T] = len_b, align_rows [B*T*L] = the pair row of
 * sentence position s: p*L2 + (s == 0 ? 0 : q_t + 1 + s) (a [PAD] row of the pair when s >= len_b), and, when
 * pair_labels [B*T, L] is not NULL, the per-type BIO labels of label_ids [B,L] (required then): for s < len_b 1 if the
 * tag is B-X_t, 2 if I-X_t, else 0; 0 for s >= len_b.  T in [1, 32] (T > 32: NER_ERR_UNSUPPORTED), L2 >= Qmax + 1 + L and
 * B*T*L2 < 2^31, else an error before any CUDA call.  One launch, no host synchronisation. */
int ner_mrc_pairs(const int32_t* token_ids, const int32_t* seq_len, const int32_t* label_ids, const int32_t* query_ids,
                  const int32_t* query_len, const int32_t* type_tag, int B, int L, int T, int Qmax, int L2, int sep_id,
                  int32_t* pair_ids, int32_t* pair_segment_ids, int32_t* pair_mask, int32_t* pair_seq_len,
                  int32_t* pair_labels, int32_t* align_rows, ner_stream_t stream);
/* The bert_mrc tag merge: logits [B*T, L, 3] f32 (O, B, I of pair p = b*T + t at sentence position s), seq_len [B],
 * type_tag [T,2] as ner_mrc_pairs -> pred_ids [B,L] i32 in the dataset's tag space.  With len_b = clamp(seq_len[b], 0, L):
 *   s >= len_b: 0;  s == 0: cls_id;  s == len_b - 1: sep_id;
 *   otherwise a_t = first argmax of type t's logits; among the types with a_t != O the one with the highest
 *   z[a_t] - logsumexp(z) (fp32) wins, the lowest t on a tie; its B-X / I-X tag id, o_id when no type claims s.
 * T in [1, 32] (T > 32: NER_ERR_UNSUPPORTED), B*T*L < 2^31.  One launch. */
int ner_mrc_merge(const float* logits, const int32_t* seq_len, const int32_t* type_tag, int B, int L, int T, int o_id,
                  int cls_id, int sep_id, int32_t* pred_ids, ner_stream_t stream);
/* model/bert_mrc_span.py: the span-pointer MRC model (Li et al., ACL 2020) over the bert_mrc pairs p = b*T + t, each with
 * the sentence-aligned rows [L, H] of ner_mrc_pairs / ner_gather_rows, len_p = clamp(pair_seq_len[p], 0, L), m_p = len_p-2.
 * Candidates are the (i, j) with 1 <= i <= j <= m_p (sentence content, no [CLS] / [SEP]).  Common rules: L <= 511, I % 32 == 0
 * and I <= 4096, T <= 32, else NER_ERR_UNSUPPORTED; P*L*L < 2^31; P = 0 / B = 0 is a no-op; every check runs before any CUDA
 * call; no allocation, no float atomics, bit-identical repeats.
 *
 * Targets from the per-type BIO labels y [P, L] of ner_mrc_pairs (0 O, 1 B, 2 I): start_y[p,s] = [s < len_p and y = 1];
 * span_end[p,s] = r(s), the last j >= s, j < len_p, with y[s+1..j] all 2, for a start s, else -1; end_y[p,j] = [j = r(s) for
 * some start s].  An I-run without a B in front gives no span.  All three [P, L] i32, fully written.  One launch. */
int ner_mrc_span_targets(const int32_t* pair_labels, const int32_t* pair_seq_len, int P, int L, int32_t* start_y,
                         int32_t* end_y, int32_t* span_end, ner_stream_t stream);
/* Match head forward.  uv [P*L, ld_uv] f32 is the projection GEMM's output as it lies: row p*L + s holds U[p,s,0:I] in
 * columns [0, I) and V[p,s,0:I] in [I, 2I) (ld_uv >= 2I, ld_uv % 4 == 0; uv, b1, w2 16-byte aligned).  b1 [I], w2 [I], b2 [1].
 *   z[p,i,j] = b2 + sum_k w2[k] * m_k / keep * GELU_tanh(U[p,i,k] + V[p,j,k] + b1[k])   (k ascending, fp32; tanh.approx)
 * with m_k = [hash3(lo(seed), hi(seed) ^ (p*L + i), j*I + k) < keep * 2^32] (common.cuh) when keep_prob < 1, else 1.
 * z [P, L, L] f32 is written everywhere: the logit at the candidates, 0 elsewhere.  loss [1] (nullable) = mean over every
 * candidate of the batch of BCE-with-logits(z, [j = span_end[p,i]]) (span_end required then), 0 without candidates; the
 * candidate count is taken on the device; per-tile partials in workspace (>= ner_mrc_span_match_fwd_workspace_bytes)
 * summed in index order.  keep_prob in (0, 1]. */
size_t ner_mrc_span_match_fwd_workspace_bytes(int P, int L);
int ner_mrc_span_match_fwd(const float* uv, int ld_uv, const float* b1, const float* w2, const float* b2,
                           const int32_t* pair_seq_len, const int32_t* span_end, int P, int L, int I, float keep_prob,
                           uint64_t seed, float* z, float* loss, void* workspace, size_t workspace_bytes, ner_stream_t stream);
/* Its backward for loss * d_loss: dz = d_loss / N * (sigmoid(z) - y) at the candidates (N the candidate count), the GELU' and
 * the dropout mask recomputed from uv, b1, w2 and the forward's (keep_prob, seed).  Writes d_uv [P*L, 2I] f32 (dU | dV, 0
 * off the candidate rows), d_b1 [I], d_w2 [I], d_b2 [1] (overwritten, not accumulated).  The sums over j, over i and over
 * the pairs have one owner each or are per-CTA partials in workspace (>= ner_mrc_span_match_bwd_workspace_bytes) added in
 * pair order.  Three launches. */
size_t ner_mrc_span_match_bwd_workspace_bytes(int P, int I);
int ner_mrc_span_match_bwd(const float* uv, int ld_uv, const float* z, const float* b1, const float* w2,
                           const int32_t* pair_seq_len, const int32_t* span_end, int P, int L, int I, float d_loss,
                           float keep_prob, uint64_t seed, float* d_uv, float* d_b1, float* d_w2, float* d_b2, void* workspace,
                           size_t workspace_bytes, ner_stream_t stream);
/* PREDICT / EVAL decode of B sentences (seq_len [B]; P = B*T pairs, pair p = b*T + t).  start_logits / end_logits [P, L, 2]
 * f32: s is a start (end) of type t when 1 <= s <= m and its two logits' first argmax is 1.  z is computed (bit-identical to
 * ner_mrc_span_match_fwd at keep 1) only for start i <= end j; a span (i, j, t) is kept when z > 0, with probability
 * sigmoid(z).  spans [B, cap] i32 = i | (j + 1) << 12 | t << 24 (ner_extract_spans' word), span_probs [B, cap] f32, ordered
 * by (start, end, type); span_counts [B] = the true count (spans past cap are dropped; slots past the count are 0).  pred_ids [B, L]:
 * the greedy non-overlapping projection of all spans of the sentence (descending z, then lower type, start, end; a span
 * overlapping a kept one is skipped), B-X_t at i and I-X_t on i+1..j by type_tag [T, 2], o_id elsewhere in 1..len-2;
 * cls_id at 0, sep_id at len - 1, 0 from len on (ner_mrc_merge's rules).  workspace >=
 * ner_mrc_span_decode_workspace_bytes(B*T, L).  cap >= 0 (spans / span_probs may be NULL when cap = 0).  Three launches. */
size_t ner_mrc_span_decode_workspace_bytes(int P, int L);
int ner_mrc_span_decode(const float* start_logits, const float* end_logits, const float* uv, int ld_uv, const float* b1,
                        const float* w2, const float* b2, const int32_t* seq_len, const int32_t* type_tag, int B, int T, int L,
                        int I, int o_id, int cls_id, int sep_id, int cap, int32_t* pred_ids, int32_t* spans,
                        float* span_probs, int32_t* span_counts, void* workspace, size_t workspace_bytes,
                        ner_stream_t stream);
/* model/bert_global_pointer.py: the GlobalPointer span head (Su, 2021; a restatement, not pinned to the reference) over the
 * BertModel sequence output of B sentences, T entity types, head size D = 64.  The projection P [rows, T*2D] f32 (one
 * GEMM) holds q of type t in columns [t*2D, t*2D + D) and k in [t*2D + D, (t+1)*2D).  Rows are addressed padded (row b*L + s,
 * cu_seqlens NULL) or packed (row cu_seqlens[b] + s, cu_seqlens [B+1] from ner_seq_pack_plan), as ner_bilstm_recurrence.
 * With len_b = clamp(seq_len[b], 0, L) and m_b = len_b - 2, the candidates are 1 <= i <= j <= m_b and
 *   s[b,t,i,j] = q'_i . k'_j,   q' = RoPE_i(q) / 8,  k' = RoPE_j(k),
 * RoPE_s rotating each pair (2i, 2i+1) by the angle s * 10000^(-2i/D).  Common rules: T in [1, 32] and L <= 512, else
 * NER_ERR_UNSUPPORTED; B*T*L*L < 2^31; B = 0 is a no-op; every check runs before any CUDA call; no allocation, no float
 * atomics, bit-identical repeats.
 *
 * Targets: label_ids [B,L] i32, type_tag [T,2] (tag ids of B-X_t, I-X_t) -> span_end [B,T,L] i32 = for a B-X_t at s < len_b
 * the end of the I-X_t run after it (s itself without one), else -1; an I-run without a B gives no span.  One launch. */
int ner_gp_targets(const int32_t* label_ids, const int32_t* seq_len, const int32_t* type_tag, int B, int T, int L,
                   int32_t* span_end, ner_stream_t stream);
/* RoPE: proj [rows, ld_proj] f32 (ld_proj >= 2*D*T, even, 8-byte aligned) -> rot_hi bf16 [rows, T, 2, D] (q' then k' of
 * each type, 16-byte aligned; the column of an element is its column in proj) and, when rot_lo is not NULL, the bf16 rest
 * rot_lo = bf16(x - rot_hi) (ner_split_bf16's rule).  The angles are computed in double.  Rows: every (b, s < L) padded,
 * every (b, s < cu[b+1] - cu[b]) packed.  One launch. */
int ner_gp_rope(const float* proj, int ld_proj, const int32_t* cu_seqlens, int B, int T, int L, void* rot_hi, void* rot_lo,
                ner_stream_t stream);
/* Its backward: d_rot [rows, T, 2, D] f32 (16-byte aligned) -> d_proj [rows, ld_dproj] f32 = the transposed rotation (and
 * the 1/8 of q), on the rows ner_gp_rope writes.  One launch. */
int ner_gp_rope_bwd(const float* d_rot, const int32_t* cu_seqlens, int B, int T, int L, float* d_proj, int ld_dproj,
                    ner_stream_t stream);
/* Loss (bert4keras' global_pointer_crossentropy): per (b, t), with (i, j) positive iff j = span_end[b,t,i],
 *   lse_neg = log(1 + sum over negative candidates e^s),  lse_pos = log(1 + sum over positive candidates e^-s),
 * loss [1] = mean over B*T of lse_neg + lse_pos (0 for a (b, t) without candidates); lse [B*T, 2] f32 receives (lse_neg,
 * lse_pos), which ner_gp_loss_bwd reads.  S = Q'K'^T on mma.sync (bf16 -> fp32); rot_lo not NULL adds hi.lo + lo.hi
 * (fp32-accurate scores).  Per-tile partials in workspace (>= ner_gp_loss_workspace_bytes) merged in index order by a
 * second launch. */
size_t ner_gp_loss_workspace_bytes(int B, int T, int L);
int ner_gp_loss_fwd(const void* rot_hi, const void* rot_lo, const int32_t* seq_len, const int32_t* cu_seqlens,
                    const int32_t* span_end, int B, int T, int L, float* loss, float* lse, void* workspace,
                    size_t workspace_bytes, ner_stream_t stream);
/* Its backward for loss * d_loss: S recomputed from rot (bf16), dS = g e^(s - lse_neg) on negatives, -g e^(-s - lse_pos) on
 * positives, 0 off the candidates, g = d_loss / (B*T); d_rot [rows, T, 2, D] f32 = (dS K' | dS^T Q') on every row of the
 * layout (0 off the candidate rows).  Two launches: one owns query tiles, one key tiles. */
int ner_gp_loss_bwd(const void* rot, const int32_t* seq_len, const int32_t* cu_seqlens, const int32_t* span_end,
                    const float* lse, int B, int T, int L, float d_loss, float* d_rot, ner_stream_t stream);
/* PREDICT / EVAL decode.  s is computed on the tensor cores (split as ner_gp_loss_fwd when rot_lo is not NULL) into the
 * workspace (>= ner_gp_decode_workspace_bytes): after the call its first B*T*L*L floats hold s[b,t,i,j] at index
 * ((b*T + t)*L + i)*L + j for every candidate (other entries are not written).  A span (i, j, t) is kept when s > 0, with
 * span_probs = sigmoid(s) (a monotone score, not a calibrated probability).  spans [B, cap] i32 = i | (j + 1) << 12 | t << 24,
 * ordered by (start, end, type); span_counts [B] = the true count (slots past the count are 0).  pred_ids [B, L] = the greedy
 * non-overlapping projection of ner_mrc_span_decode (descending s, then lower type, start, end), with its tag rules.  cap >= 0
 * (spans / span_probs may be NULL when cap = 0).  Two launches, no host synchronisation. */
size_t ner_gp_decode_workspace_bytes(int B, int T, int L);
int ner_gp_decode(const void* rot_hi, const void* rot_lo, const int32_t* seq_len, const int32_t* cu_seqlens,
                  const int32_t* type_tag, int B, int T, int L, int o_id, int cls_id, int sep_id, int cap, int32_t* pred_ids,
                  int32_t* spans, float* span_probs, int32_t* span_counts, void* workspace, size_t workspace_bytes,
                  ner_stream_t stream);
/* Window plan of the BERT plugins' document mode (documents longer than the position table).  Document b of the [B,L]
 * batch has n_b = clamp(seq_len[b], 0, L) tokens ([CLS] ... [SEP]), m = n_b - 2 content tokens; C = W - 2.
 *   n_b = 0: no window;  n_b <= W: one window, the document itself (its rows past n_b are [PAD]);
 *   n_b > W: nw_b = 1 + ceil((m - C) / S) windows; window k starts at content offset a_k = min(k*S, m - C) and holds doc
 *   positions 0, 1 + a_k ... a_k + C, n_b - 1 (W tokens).
 * Windows are numbered document by document.  win_ids / win_segment_ids / win_mask [NW, W] i32 get the gathered
 * token_ids / segment_ids (segment_ids may be NULL: zeros) and a prefix mask; rows past the plan's windows are zero.
 * Owner of doc position t: row 0 of window 0 for t = 0, row W - 1 of the last window for t = n_b - 1; content index
 * c = t - 1 goes to the window with a_k <= c < a_k + C maximising min(c - a_k, a_k + C - 1 - c), the lowest k on a tie.
 * doc_src_padded [sum n_b] (nullable) = w*W + p of the owner (window w, row p), doc_src_packed [sum n_b] (nullable) = the
 * owner's row in the window-packed layout (windows back to back, n_b rows for a one-window document, W otherwise); both
 * indexed by the document's packed order (documents back to back, n_b rows each).
 * NW must be sum_b nw_b (windows past NW are not written).  No output may alias another output or an input.
 * W >= 3, 1 <= S <= W - 2, B, NW >= 0, L >= 1 and null token_ids / seq_len / window outputs are NER_ERR_INVALID_ARG;
 * NW*W or B*L >= 2^31 is NER_ERR_UNSUPPORTED; all before any CUDA call.  One launch, no atomics, bit-identical repeats. */
int ner_window_plan(const int32_t* token_ids, const int32_t* segment_ids, const int32_t* seq_len, int B, int L, int W, int S,
                    int NW, int32_t* win_ids, int32_t* win_segment_ids, int32_t* win_mask, int32_t* doc_src_packed,
                    int32_t* doc_src_padded, ner_stream_t stream);
/* dst[i] += a * src[i]. */
int ner_axpy_f32(float* dst, const float* src, size_t n, float a, ner_stream_t stream);
/* out[0] += sum(g^2)  (tf.clip_by_global_norm, tools/train_utils.py:315).  Deterministic (no float atomics): per-CTA partial
 * sums go to `scratch` (>= ner_sumsq_scratch_floats() floats) and are added in index order, so identical gradients give a
 * bit-identical norm on every data-parallel rank and in every run. */
size_t ner_sumsq_scratch_floats(void);
int ner_sumsq_add(const float* g, size_t n, float* out, float* scratch, ner_stream_t stream);
/* One optimizer step over a flat parameter buffer.
 * mode 0 = AdamWeightDecayOptimizer (bert optimization.py; tools/train_utils.py:276-282):
 *   g *= grad_scale * clip / max(sqrt(*gnorm_sq) * grad_scale, clip)  (gnorm_sq NULL / clip 0: no clip);
 *   m = b1 m + (1-b1) g; v = b2 v + (1-b2) g^2; p -= lr * (m / (sqrt(v) + eps) + weight_decay * p).
 * mode 1 = tf.train.AdamOptimizer (tools/train_utils.py:340-350,365-390): g clipped to
 *   [-clip, clip] (clip 0: none), p -= lr * m / (sqrt(v) + eps) with lr the bias-corrected step
 *   lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t) computed by the caller. */
int ner_adam_step(float* p, const float* g, float* m, float* v, size_t n, float lr, float beta1,
                  float beta2, float eps, float weight_decay, int mode, float clip,
                  const float* gnorm_sq, float grad_scale, ner_stream_t stream);

/* ---- encoder backward (gradient of BertModel, tools/train_utils.py:314) ---- */

/* Backward of ner_layernorm: z = y (+ residual) is recomputed from the saved operands.
 * dz = dL/dz written as f32 (residual-branch gradient) and/or bf16 (A operand of the next dgrad
 * GEMM); d_gamma / d_beta [H] are accumulated into (caller zeroes). */
int ner_layernorm_bwd(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                      const float* d_out, float* dz_f32, void* dz_bf16, float* d_gamma,
                      float* d_beta, int M, int H, float eps, ner_stream_t stream);
/* Backward of ner_layernorm_dropout: y is the UNdropped forward input; dz_f32 = gradient of the residual
 * branch, dz_bf16 = gradient w.r.t. y (masked like the forward). */
int ner_layernorm_dropout_bwd(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                              const float* d_out, float* dz_f32, void* dz_bf16, float* d_gamma,
                              float* d_beta, int M, int H, float eps, float keep_prob, uint64_t seed,
                              ner_stream_t stream);
/* Same, and additionally d_bias[H] += column sums of the (masked) dense-branch gradient — the bias gradient of the dense
 * layer whose output this LayerNorm normalises — so the separate column-sum pass over dz_bf16 is not needed.  d_bias NULL =
 * ner_layernorm_dropout_bwd. */
int ner_layernorm_dropout_bwd_bias(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                                   const float* d_out, float* dz_f32, void* dz_bf16, float* d_gamma, float* d_beta,
                                   float* d_bias, int M, int H, float eps, float keep_prob, uint64_t seed,
                                   ner_stream_t stream);
/* bf16 [M,N] -> bf16 [N,Mp] zero padded (K-major operands of weight-gradient GEMMs). */
int ner_transpose_bf16(const void* src_bf16, void* dst_bf16, int M, int N, int Mp,
                       ner_stream_t stream);
/* out[n] += sum_m x[m,n], x bf16 [M,N]  (bias gradients). */
int ner_colsum_bf16_add(const void* x_bf16, float* out, int M, int N, ner_stream_t stream);
/* GELU on a saved bf16 pre-activation (training forward) and its backward d_pre = d_act * gelu'(pre).
 * n % 4 == 0.  erf_variant: 0 tanh approximation, 1 erf. */
int ner_gelu_bf16(const void* pre_bf16, void* act_bf16, size_t n, int erf_variant, ner_stream_t stream);
/* Same on f32 (exact tanhf / erff): the FFN activation of the fp32-accurate BERT mode (y may alias x). */
int ner_gelu_f32(const float* x, float* y, size_t n, int erf_variant, ner_stream_t stream);
int ner_gelu_bwd_bf16(const void* pre_bf16, const void* dact_bf16, void* dpre_bf16, size_t n,
                      int erf_variant, ner_stream_t stream);
/* GELU backward on [M, N] with the bias gradient of the dense layer in front of the GELU fused in:
 * d_pre = d_act * gelu'(pre) and d_bias[N] += column sums of (the bf16-rounded) d_pre.  N % 8 == 0. */
int ner_gelu_bwd_bias_bf16(const void* pre_bf16, const void* dact_bf16, void* dpre_bf16, float* d_bias, int M, int N,
                           int erf_variant, ner_stream_t stream);
/* Embedding backward: scatter-add dx [B*L,H] f32 into d_word [vocab,H], d_type [n_type,H],
 * d_pos [>=L,H] (all accumulated into). */
int ner_bert_embed_bwd(const float* dx, const int32_t* ids, const int32_t* seg, float* d_word,
                       float* d_type, float* d_pos, int B, int L, int H, int vocab, int n_type,
                       ner_stream_t stream);
/* Backward of ner_bert_attention (padded layout, head_dim 64): qkv / ctx from the forward pass,
 * dctx = dL/dctx; writes d_qkv (bf16, layout of qkv).  Scores are recomputed, nothing L x L is stored;
 * (keep_prob, seed) must be the forward call's so the dropout mask is regenerated.  Any L: above 384 the kernels tile
 * the keys and keep per-row statistics in d_qkv between launches, so d_qkv must not alias qkv, ctx or dctx. */
int ner_bert_attention_bwd(const void* qkv_bf16, const int32_t* mask, const void* ctx_bf16,
                           const void* dctx_bf16, void* dqkv_bf16, int B, int L, int num_heads,
                           int head_dim, float scale, float mask_add, float keep_prob, uint64_t seed,
                           ner_stream_t stream);
/* Packed layout: sequence b occupies rows [cu_seqlens[b], cu_seqlens[b+1]) of qkv / ctx / dctx / dqkv, every key valid;
 * L is the longest sequence.  Rows of dqkv past cu_seqlens[B] are not touched; dqkv must not alias qkv, ctx or dctx. */
int ner_bert_attention_bwd_packed(const void* qkv_bf16, const int32_t* cu_seqlens, const void* ctx_bf16,
                                  const void* dctx_bf16, void* dqkv_bf16, int B, int L, int num_heads,
                                  int head_dim, float scale, float keep_prob, uint64_t seed,
                                  ner_stream_t stream);

/* Weight gradients of several dense layers in ONE launch (tools/train_utils.py:314 `tf.gradients` w.r.t. the dense kernels):
 *   dw_p[k_in, n_out] (f32, accumulated into) += x_p^T . dy_p[:, dy_col0 : dy_col0 + n_out]
 * x_p bf16 [rows, ld_x] (the layer's input activations, first k_in columns used), dy_p bf16 [rows, ld_dy] (gradient w.r.t. the
 * layer's output).  Both are consumed as they lie (token-major = MN-major wgmma operands, 64 x 64 TMA boxes): no transposed
 * copies.  k_in % 128 == 0, n_out % 256 == 0, dy_col0 % 64 == 0, ld % 8 == 0; at most 6 problems per call. */
typedef struct {
  const void* x_bf16;
  int ld_x;
  const void* dy_bf16;
  int ld_dy;
  int dy_col0;
  float* dw;
  int k_in;
  int n_out;
} ner_wgrad_problem;
int ner_wgrad_group_bf16(const ner_wgrad_problem* problems_host, int count, int rows, ner_stream_t stream);

/* Data-parallel overlap hook (SURVEY 8e; no reference counterpart — the reference is single device): events_host[l]
 * (cudaEvent_t, HOST array of n_events handles, NULL entries skipped) is recorded on the stream of the NEXT
 * ner_bert_encoder_train_bwd / _bwd_packed calls of this host thread as soon as every gradient of encoder layer l is
 * enqueued, so the caller can all-reduce that layer's slice of the flat gradient buffer while the backward pass of the
 * layers below still runs.  n_events = 0 clears the hook. */
int ner_bert_train_bwd_set_layer_events(void* const* events_host, int n_events);

/* tools/infer_utils.py:76-99  extract_entity — the tag-sequence half of it, on the device: pred_ids [B,L] i32 ->
 * per sentence the entity spans in order.  tag_class [K] u8 describes idx2tag: bits 0-1 kind (0 other, 1 'B', 2 'I' by
 * tag.split('-')[0]), bit 2 = the tag's first character is 'B' or 'I' (the reference's test on the previous tag),
 * bits 3-7 entity type id (index of tag.split('-')[1] in the caller's type list).  spans [B,cap] i32, each
 * start | end << 12 | type << 24 with end exclusive; counts [B] i32 = spans found (may exceed cap: the rest is dropped).
 * Reproduces the reference scan exactly, including its treatment of ill-formed sequences (an I after an I opens a span,
 * a span is typed by its LAST tag).  L <= 4095. */
int ner_extract_spans(const int32_t* pred_ids, const uint8_t* tag_class, int32_t* spans, int32_t* counts, int B, int L,
                      int K, int cap, ner_stream_t stream);
/* ner_extract_spans for tag sets of more than 32 entity types: tag_class [K] u16 with the same bits 0-2 and the type id
 * in bits 3-9 (up to 128 types); the span word carries it in bits 24-30. */
int ner_extract_spans_wide(const int32_t* pred_ids, const uint16_t* tag_class, int32_t* spans, int32_t* counts, int B,
                           int L, int K, int cap, ner_stream_t stream);

/* ------------------------------------------------------------------------ *
 * Raw text -> BasicProc.build_seq_feature features (data/device_featurize.py builds the tables).
 * text: the B texts' UTF-8 bytes (Python's encode('utf-8', 'surrogatepass')) back to back, text b =
 * [offsets[b], offsets[b+1]); offsets [B+1] i64 on the device and the same values in host memory (offsets_host), which
 * is checked: offsets_host[0] == 0 and non-decreasing.  Malformed UTF-8 reads as U+FFFD.
 * Unicode tables: uni_stage2[(uni_stage1[cp >> 8] << 8) + (cp & 255)] u32 = flags (bit 0 _is_control, 1 _is_whitespace,
 * 2 str.isspace, 3 _is_punctuation, 4 _is_chinese_char, 5 category Mn, 6 cased and not case-ignorable, 7
 * case-ignorable) | combining class << 8 | x << 16, where x > 0 names NFD(lower(cp)) = uni_expand[4x .. 4x+3] (zero
 * padded) and x = 0 means cp itself.
 * Vocabulary: open addressing over the UTF-8 bytes of every key (FNV-1a 32, linear probing): slots [n_slots] i32 (a
 * power of two, -1 = empty) -> entry e; entries [n_keys, 3] i32 = blob offset, byte length, id; blob = the keys' bytes.
 * Outputs [B, L] i32 token_ids / mask / segment_ids / unk_cursor and seq_len [B] i32.  One launch, no host
 * synchronisation, shared memory independent of the texts' length; a row stops scanning once it is full.
 * NER_ERR_INVALID_ARG for B < 0, L < 1 (L < 2 for WordPiece), a null pointer, bad offsets, n_slots not a power of two, a
 * negative special id or max_piece < 1; NER_ERR_UNSUPPORTED for B*L >= 2^31; all before any CUDA call.  B = 0 is a
 * no-op. */
/* FullTokenizer.tokenize (BasicTokenizer(do_lower_case) + WordPiece, 200-character [UNK] rule) + format_sequence:
 * [CLS] + the first L-2 tokens + [SEP], then [PAD].  Token ids must be below 2^24; max_piece = the longest key in code
 * points.  unk_cursor = fix_tokens' cursor at each [UNK] (characters of the tokens before it, '##' removed, an [UNK]
 * counting one), -1 elsewhere. */
int ner_featurize_wordpiece(const uint8_t* text, const int64_t* offsets, const int64_t* offsets_host, int B, int L,
                            const uint16_t* uni_stage1, const uint32_t* uni_stage2, const uint32_t* uni_expand,
                            const int32_t* slots, int n_slots, const int32_t* entries, const uint8_t* blob,
                            int max_piece, int do_lower_case, int cls_id, int sep_id, int pad_id, int unk_id,
                            int32_t* token_ids, int32_t* mask, int32_t* segment_ids, int32_t* seq_len,
                            int32_t* unk_cursor, ner_stream_t stream);
/* TokenizerAdapter.tokenize + format_sequence: characters for which str.strip() is empty are skipped, full2half, the
 * character's id or unk_id, the first L tokens, then pad_id.  unk_cursor = the raw character index of each [UNK]. */
int ner_featurize_chars(const uint8_t* text, const int64_t* offsets, const int64_t* offsets_host, int B, int L,
                        const uint16_t* uni_stage1, const uint32_t* uni_stage2, const int32_t* slots, int n_slots,
                        const int32_t* entries, const uint8_t* blob, int pad_id, int unk_id, int32_t* token_ids,
                        int32_t* mask, int32_t* segment_ids, int32_t* seq_len, int32_t* unk_cursor,
                        ner_stream_t stream);

/* ------------------------------------------------------------------------ *
 * SoftLexicon HOST builder — replaces data/word_enhance.py:302-337 (build_soft_lexicon), :89-119 (align_with_token),
 * :163-205 (postproc_soft_lexicon) and data/base_preprocess.py:397-412 (format_soft_seq) for whole datasets at a time.
 * Host code (no CUDA call, no stream): all pointers are HOST pointers.  Output layout = the input of
 * ner_softlexicon_pool_fwd: [n_sent, max_seq_len, 4 (B,M,E,S), 10] ids / weights.
 * ------------------------------------------------------------------------ */
typedef struct ner_lexicon ner_lexicon;
/* Trie over the word vocabulary.  Words are UTF-32 code points back to back, word w = [offsets[w], offsets[w+1]); its id
 * is w (= embedding row).  freq[n_words + 2]: per-word frequency, then <None> (id n_words, reference: 1) and <PAD>
 * (id n_words + 1, reference: 0) — VocabModel._addon_token, data/word_enhance.py:62-70.  NULL on bad input. */
ner_lexicon* ner_lexicon_create(const uint32_t* word_codepoints_host, const int64_t* word_offsets_host,
                                const double* freq_host, int n_words);
void ner_lexicon_destroy(ner_lexicon* lexicon);
int64_t ner_lexicon_num_nodes(const ner_lexicon* lexicon);
/* Sentences are UTF-32 code points (spaces already removed, as build_soft_lexicon does), sentence s =
 * [sent_offsets[s], sent_offsets[s+1]).  tok_len / tok_offsets (both NULL, or per sentence the number of characters
 * each token covers, for WordPiece tokenizers): rows of characters one token swallowed are merged by set union.
 * bert_mode != 0: row 0 ([CLS]) and the rows from the [SEP] on stay zero and at most max_seq_len - 2 tokens are kept.
 * Every set holds its matches in first-seen order (the reference iterates Python sets: unordered), an empty set holds
 * <None>, sets are padded with <PAD> to 10 or cut to the 10 most frequent (stable), weights = freq / sum over the
 * token's 40 slots.  n_threads <= 0: one per hardware thread.  ids_out / weights_out: [n_sent, max_seq_len * 40]. */
int ner_lexicon_build(const ner_lexicon* lexicon, const uint32_t* codepoints_host, const int64_t* sent_offsets_host,
                      int n_sent, const int32_t* tok_len_host, const int64_t* tok_offsets_host, int max_seq_len,
                      int bert_mode, int32_t* ids_out_host, float* weights_out_host, int n_threads);
/* Lattice word lists of the lattice_lstm_crf plugin (giga characters only), same trie walk and thread pool as
 * ner_lexicon_build.  For each start character b < max_seq_len, the vocabulary words of 2..10 characters that match the
 * sentence at [b, b + n) fill the Kw slots [b * Kw, (b + 1) * Kw): at most Kw of them, the most frequent first (stable
 * over the trie's discovery order, i.e. increasing length).  A word must end inside the first max_seq_len characters.
 * Empty slots: id <PAD> (n_words + 1), length 0.  ids_out / lens_out: [n_sent, max_seq_len * Kw] int32.
 * dropped_out (may be NULL): number of matches the Kw cap discarded over all sentences.  1 <= Kw <= 8. */
int ner_lexicon_build_lattice(const ner_lexicon* lexicon, const uint32_t* codepoints_host, const int64_t* sent_offsets_host,
                              int n_sent, int max_seq_len, int Kw, int32_t* ids_out_host, int32_t* lens_out_host,
                              int64_t* dropped_out_host, int n_threads);

/* ------------------------------------------------------------------------ *
 * Lattice LSTM recurrence (Zhang & Yang, ACL 2018) — model/lattice_lstm_crf.py.  Padded layout [B, L].
 * ------------------------------------------------------------------------ */
/* Word slots: lat_len [B, L * Kw] int32, slot (b, p, k) = a word of lat_len characters starting at position p.  A slot is
 * empty when its length is outside [2, 10] or the word would reach past seq_len[b].  Per direction d (fw = 0, bw = 1):
 *   xproj [B*L, 8H]: columns d*4H + (z_i, z_o, z_g, x-part of alpha) = x_t W + b of the char cell and alpha;
 *   wproj [B*L*Kw, 6H]: columns d*3H + (z_f, z_i, z_g) = x^w W_x + b of the word cell of slot (b, p, k);
 *   wrec_d [H, 6H] = [char_cell kernel[Ec:] | word_cell kernel[Ew:]];  wac_d [H, H] = alpha kernel[Ec:].
 * out [B, L, 2H] (fw | bw, zero for t >= seq_len).  The backward direction runs right to left and merges a word at its
 * first character; its cell is computed at the word's last character.  Training saves (all NULL or all given):
 *   gates [B*L, 6H] (sigmoid i, sigmoid o, tanh g per direction), cstate [B, L, 2H], norm [B, L, 2H] (e^i + sum e^a, 0 at
 *   steps without words), wgates [B*L*Kw, 6H] (sigmoid f, sigmoid i, tanh g), cw / aw / hw [B*L*Kw, 2H] (word cell,
 *   alpha gate, h the word cell read).  Slot outputs are written for filled slots only: the caller zeroes them.
 * Limits: Kw <= 8; H small enough for the recurrent weights to fit on a cluster of at most 8 CTAs (H <= 240). */
int ner_lattice_recurrence(const float* xproj, const float* wproj, const int32_t* lat_len, const float* wrec_fw,
                           const float* wrec_bw, const float* wac_fw, const float* wac_bw, const int32_t* seq_len,
                           float* out, int B, int L, int H, int Kw, float* gates, float* cstate, float* norm,
                           float* wgates, float* cw, float* aw, float* hw, ner_stream_t stream);
/* Back-propagation through time of ner_lattice_recurrence, from its saved tensors.  Writes d_xproj [B*L, 8H] (every row;
 * zero for t >= seq_len), and for filled slots only d_wproj [B*L*Kw, 6H] and d_alpha [B*L*Kw, 2H] (the gradient of the
 * alpha pre-activation of each word): the caller zeroes those two.  Weight gradients are GEMMs over them:
 * dW_rec = [h_prev^T dz_char | hw^T d_wproj], dW_ac = cw^T d_alpha, dW_x = x^T d_xproj, d_bias = column sums. */
int ner_lattice_recurrence_bwd(const float* d_out, const float* gates, const float* cstate, const float* norm,
                               const float* wgates, const float* cw, const float* aw, const int32_t* lat_len,
                               const float* wrec_fw, const float* wrec_bw, const float* wac_fw, const float* wac_bw,
                               const int32_t* seq_len, float* d_xproj, float* d_wproj, float* d_alpha, int B, int L,
                               int H, int Kw, ner_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* NER_B200_H_ */
