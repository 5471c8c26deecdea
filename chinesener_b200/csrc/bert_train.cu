// TRAIN-mode BertModel forward and backward as two C-ABI calls (bert_base.bert.modeling.BertModel
// with is_training=True as driven from reference tools/layer.py:63-81, gradients as tf.gradients
// derives them at tools/train_utils.py:314).  The host loops below only enqueue kernels (≈11 per
// layer forward, ≈27 per layer backward) on the caller's stream: issued from Python the same
// sequence costs tens of microseconds of host time per launch, which made the TRAIN step launch-bound.
//
// Saved activations (padded layout, rows = B*L), one block per layer:
//   x32 f32 | x16 bf16 (layer input) | qkv bf16 | ctx bf16 | y1 bf16 | x1_32 f32 | x1_16 bf16 |
//   pre bf16 | inter bf16 | y2 bf16   (y1 / y2 are kept UNdropped: the LayerNorm kernels apply the hidden dropout);    the encoder output is the caller's out_f32 / out_bf16.
// Dropout seeds: every site draws seed = base + index (embedding 0; layer l: 1+3l attention probs,
// 2+3l attention-output dense, 3+3l FFN-output dense); the backward call regenerates the masks.
#include <vector>

#include "common.cuh"

namespace {

inline size_t al(size_t x) { return (x + 255) & ~(size_t)255; }

struct LayerSaved {
  float* x32;
  void* x16;
  void* qkv;
  void* ctx;
  void* y1;
  float* x1_32;
  void* x1_16;
  void* pre;
  void* inter;
  void* y2;
};

size_t layer_saved_bytes(size_t R, size_t H, size_t I) {
  return al(R * H * 4) + al(R * H * 2) + al(R * 3 * H * 2) + al(R * H * 2) + al(R * H * 2) + al(R * H * 4) + al(R * H * 2) +
         al(R * I * 2) + al(R * I * 2) + al(R * H * 2);
}

LayerSaved carve(uint8_t* p, size_t R, size_t H, size_t I) {
  LayerSaved s;
  s.x32 = reinterpret_cast<float*>(p);   p += al(R * H * 4);
  s.x16 = p;                             p += al(R * H * 2);
  s.qkv = p;                             p += al(R * 3 * H * 2);
  s.ctx = p;                             p += al(R * H * 2);
  s.y1 = p;                              p += al(R * H * 2);
  s.x1_32 = reinterpret_cast<float*>(p); p += al(R * H * 4);
  s.x1_16 = p;                           p += al(R * H * 2);
  s.pre = p;                             p += al(R * I * 2);
  s.inter = p;                           p += al(R * I * 2);
  s.y2 = p;
  return s;
}

#define NER_TRY(call)              \
  do {                             \
    const int rc_ = (call);        \
    if (rc_ != NER_OK) return rc_; \
  } while (0)

// dW [K_in, N_out] f32 += x^T · dy   (x [R, K_in], dy [R, N_out] bf16): both operands transposed to K-major
// (K = tokens) and multiplied on the tensor cores with the accumulate-into-residual epilogue.
int wgrad(const void* x, int k_in, const void* dy_t /* [N_out, Rp] or null */, const void* dy, int n_out, float* dw, int R,
          int Rp, void* xt, void* dyt, cudaStream_t st) {
  NER_TRY(ner_transpose_bf16(x, xt, R, k_in, Rp, st));
  const void* b = dy_t;
  if (b == nullptr) {
    NER_TRY(ner_transpose_bf16(dy, dyt, R, n_out, Rp, st));
    b = dyt;
  }
  return ner_gemm_bf16(xt, b, nullptr, dw, dw, k_in, n_out, Rp, NER_EPI_RES_F32, 0, st);
}

// dq[m, n] += t[m, n], dk[m, n] += t[m, H + n], dv[m, n] += t[m, 2H + n]   (t [H, 3H] f32, H % 4 == 0)
__global__ void __launch_bounds__(256)
add_split3_kernel(const float* __restrict__ t, float* __restrict__ dq, float* __restrict__ dk, float* __restrict__ dv, int H) {
  const int hv = H / 4;
  const size_t total = (size_t)H * 3 * hv, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t m = i / (3 * hv), c = i - m * (3 * hv);
    const int j = (int)(c / hv), n4 = (int)(c - (size_t)j * hv);
    float* dst = (j == 0 ? dq : (j == 1 ? dk : dv)) + m * H + (size_t)n4 * 4;
    const float4 a = *reinterpret_cast<const float4*>(t + m * 3 * H + (size_t)j * H + (size_t)n4 * 4);
    float4 d = *reinterpret_cast<float4*>(dst);
    d.x += a.x; d.y += a.y; d.z += a.z; d.w += a.w;
    *reinterpret_cast<float4*>(dst) = d;
  }
}

}  // namespace

extern "C" size_t ner_bert_train_saved_bytes(const ner_bert_config* cfg, int rows) {
  if (!cfg || rows < 0) return 0;
  const size_t R = (size_t)rows, H = (size_t)cfg->hidden_size, I = (size_t)cfg->intermediate_size;
  return (size_t)cfg->num_layers * layer_saved_bytes(R, H, I) + al(R * H * 4) /* embedding sum */;
}

extern "C" size_t ner_bert_train_packed_saved_bytes(const ner_bert_config* cfg, int n_packed) {
  if (!cfg || n_packed < 0) return 0;
  const size_t R = (size_t)n_packed, H = (size_t)cfg->hidden_size;
  return ner_bert_train_saved_bytes(cfg, n_packed) + al(R * H * 4) + al(R * H * 2) /* packed encoder output */;
}

extern "C" size_t ner_bert_train_packed_scratch_bytes(const ner_bert_config* cfg, int n_packed, int padded_rows) {
  if (!cfg || n_packed < 0 || padded_rows < n_packed) return 0;
  return ner_bert_train_scratch_bytes(cfg, n_packed) + al((size_t)padded_rows * cfg->hidden_size * 4) /* padded d_embedding */;
}

extern "C" size_t ner_bert_train_scratch_bytes(const ner_bert_config* cfg, int rows) {
  if (!cfg || rows < 0) return 0;
  const size_t R = (size_t)rows, Rp = (R + 7) / 8 * 8, H = (size_t)cfg->hidden_size, I = (size_t)cfg->intermediate_size;
  const size_t W = I > 3 * H ? I : 3 * H;
  return 2 * al(R * H * 4)      // d ping-pong (f32)
         + al(R * H * 4)        // dz f32 (residual-path gradient)
         + 2 * al(R * H * 2)    // dz bf16 of the two LayerNorm backward passes (both live until the layer's grouped wgrad launch)
         + 2 * al(R * I * 2)    // dinter, dpre
         + al(R * H * 2)        // dctx
         + al(R * 3 * H * 2)    // dqkv
         + 2 * al(W * Rp * 2)   // transposed operands of the weight-gradient GEMMs
         + al(3 * H * 4)        // fused QKV bias gradient
         + al(3 * H * H * 4);   // fused QKV weight gradient [H, 3H] f32
}

// Packed mode (cu_seqlens / tok_src / n_packed from ner_seq_pack_plan): every per-token kernel runs on the n_packed real
// tokens only and the attention kernels take cu_seqlens; the padded <-> packed row moves happen once at each end
// (embedding sum in, encoder output out; d_out in, embedding gradient out).  [PAD] rows of the output are zero.
static int train_fwd_impl(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                          const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                          const ner_bert_layer_weights* layers, const int32_t* ids, const int32_t* mask,
                          const int32_t* seg, int B, int L, const int32_t* cu_seqlens, const int32_t* tok_src, int n_packed,
                          float hidden_keep, float attn_keep,
                          uint64_t seed, float* out_f32, void* out_bf16, void* saved, size_t saved_bytes,
                          ner_stream_t stream) {
  const bool packed = cu_seqlens != nullptr;
  if (!cfg || !layers || !out_f32 || !out_bf16 || !ids || (!mask && !packed) || !saved) return NER_ERR_INVALID_ARG;
  if (B < 0 || L < 1 || !(hidden_keep > 0.f) || hidden_keep > 1.f || !(attn_keep > 0.f) || attn_keep > 1.f)
    return NER_ERR_INVALID_ARG;
  if (packed && (!tok_src || n_packed < 0 || n_packed > B * L)) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  const int rows = packed ? n_packed : B * L, H = cfg->hidden_size, NH = cfg->num_heads, I = cfg->intermediate_size;
  if (H % NH != 0) return NER_ERR_INVALID_ARG;
  if (saved_bytes < (packed ? ner_bert_train_packed_saved_bytes(cfg, rows) : ner_bert_train_saved_bytes(cfg, rows)))
    return NER_ERR_WORKSPACE;
  cudaStream_t cst = static_cast<cudaStream_t>(stream);
  if (packed) {
    if (cudaMemsetAsync(out_f32, 0, (size_t)B * L * H * 4, cst) != cudaSuccess) return NER_ERR_CUDA_BASE - (int)cudaGetLastError();
    if (cudaMemsetAsync(out_bf16, 0, (size_t)B * L * H * 2, cst) != cudaSuccess) return NER_ERR_CUDA_BASE - (int)cudaGetLastError();
    if (rows == 0) return NER_OK;
  }
  const size_t R = (size_t)rows, lb = layer_saved_bytes(R, H, I);
  uint8_t* base = static_cast<uint8_t*>(saved);
  float* emb_sum = reinterpret_cast<float*>(base + (size_t)cfg->num_layers * lb);
  float* last32 = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(emb_sum) + al(R * H * 4));   // packed mode only
  void* last16 = reinterpret_cast<uint8_t*>(last32) + al(R * H * 4);
  const int gelu_erf = cfg->gelu_erf ? 1 : 0;
  const float scale = 1.0f / sqrtf((float)(H / NH));

  // embeddings: sum -> LayerNorm -> dropout   (layer_norm_and_dropout of embedding_postprocessor)
  LayerSaved s0 = carve(base, R, H, I);
  if (packed) {   // padded sum staged in the caller's (still unused) output buffer, real rows gathered out of it
    NER_TRY(ner_bert_embed_sum(word_emb, type_emb, pos_emb, ids, seg, out_f32, B, L, H, cfg->vocab_size, cfg->type_vocab_size,
                               cfg->max_position, stream));
    NER_TRY(ner_gather_rows(out_f32, tok_src, emb_sum, rows, H * 4, stream));
    if (cudaMemsetAsync(out_f32, 0, (size_t)B * L * H * 4, cst) != cudaSuccess) return NER_ERR_CUDA_BASE - (int)cudaGetLastError();
  } else
  NER_TRY(ner_bert_embed_sum(word_emb, type_emb, pos_emb, ids, seg, emb_sum, B, L, H, cfg->vocab_size, cfg->type_vocab_size,
                             cfg->max_position, stream));
  NER_TRY(ner_layernorm(emb_sum, 0, nullptr, emb_ln_gamma, emb_ln_beta, s0.x32, s0.x16, rows, H, cfg->ln_eps, stream));
  if (hidden_keep < 1.f) {
    NER_TRY(ner_dropout(s0.x32, s0.x32, R * H, hidden_keep, seed, stream));
    NER_TRY(ner_cast_bf16(s0.x32, s0.x16, R * H, stream));
  }
  for (int l = 0; l < cfg->num_layers; ++l) {
    const ner_bert_layer_weights& w = layers[l];
    LayerSaved s = carve(base + (size_t)l * lb, R, H, I);
    const bool last = l + 1 == cfg->num_layers;
    LayerSaved nx = last ? s : carve(base + (size_t)(l + 1) * lb, R, H, I);
    float* o32 = last ? (packed ? last32 : out_f32) : nx.x32;
    void* o16 = last ? (packed ? last16 : out_bf16) : nx.x16;
    const uint64_t sa = seed + 1 + 3 * (uint64_t)l, s1 = sa + 1, s2 = sa + 2;
    NER_TRY(ner_gemm_bf16(s.x16, w.wqkv, w.bqkv, nullptr, s.qkv, rows, 3 * H, H, NER_EPI_BF16, 0, stream));
    NER_TRY(ner_bert_attention(s.qkv, mask, s.ctx, B, L, NH, H / NH, scale, -10000.0f, cu_seqlens, rows, attn_keep, sa, stream));
    NER_TRY(ner_gemm_bf16(s.ctx, w.wo, w.bo, nullptr, s.y1, rows, H, H, NER_EPI_BF16, 0, stream));
    NER_TRY(ner_layernorm_dropout(s.y1, 1, s.x32, w.ln1_gamma, w.ln1_beta, s.x1_32, s.x1_16, rows, H, cfg->ln_eps, hidden_keep, s1,
                                  stream));
    NER_TRY(ner_gemm_bf16(s.x1_16, w.wi, w.bi, nullptr, s.pre, rows, I, H, NER_EPI_BF16, 0, stream));
    NER_TRY(ner_gelu_bf16(s.pre, s.inter, R * I, gelu_erf, stream));
    NER_TRY(ner_gemm_bf16(s.inter, w.wd, w.bd, nullptr, s.y2, rows, H, I, NER_EPI_BF16, 0, stream));
    NER_TRY(ner_layernorm_dropout(s.y2, 1, s.x1_32, w.ln2_gamma, w.ln2_beta, o32, o16, rows, H, cfg->ln_eps, hidden_keep, s2,
                                  stream));
  }
  if (packed) {
    NER_TRY(ner_scatter_rows(last32, tok_src, out_f32, rows, H * 4, stream));
    NER_TRY(ner_scatter_rows(last16, tok_src, out_bf16, rows, H * 2, stream));
  }
  return NER_OK;
}

extern "C" int ner_bert_encoder_train_fwd(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                                          const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                                          const ner_bert_layer_weights* layers, const int32_t* ids, const int32_t* mask,
                                          const int32_t* seg, int B, int L, float hidden_keep, float attn_keep,
                                          uint64_t seed, float* out_f32, void* out_bf16, void* saved, size_t saved_bytes,
                                          ner_stream_t stream) {
  if (!mask) return NER_ERR_INVALID_ARG;
  return train_fwd_impl(cfg, word_emb, type_emb, pos_emb, emb_ln_gamma, emb_ln_beta, layers, ids, mask, seg, B, L, nullptr, nullptr,
                        0, hidden_keep, attn_keep, seed, out_f32, out_bf16, saved, saved_bytes, stream);
}

extern "C" int ner_bert_encoder_train_fwd_packed(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                                                 const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                                                 const ner_bert_layer_weights* layers, const int32_t* ids, const int32_t* seg,
                                                 int B, int L, const int32_t* cu_seqlens, const int32_t* tok_src, int n_packed,
                                                 float hidden_keep, float attn_keep, uint64_t seed, float* out_f32,
                                                 void* out_bf16, void* saved, size_t saved_bytes, ner_stream_t stream) {
  if (!cu_seqlens) return NER_ERR_INVALID_ARG;
  return train_fwd_impl(cfg, word_emb, type_emb, pos_emb, emb_ln_gamma, emb_ln_beta, layers, ids, nullptr, seg, B, L, cu_seqlens,
                        tok_src, n_packed, hidden_keep, attn_keep, seed, out_f32, out_bf16, saved, saved_bytes, stream);
}

// Optional per-layer completion events of the backward composites (data-parallel gradient exchange overlapped with the
// backward pass): events[l] is recorded on the composite's stream once every gradient of encoder layer l has been enqueued.
static thread_local std::vector<cudaEvent_t> tl_layer_events;

extern "C" int ner_bert_train_bwd_set_layer_events(void* const* events_host, int n_events) {
  if (n_events < 0 || (n_events > 0 && !events_host)) return NER_ERR_INVALID_ARG;
  tl_layer_events.assign(reinterpret_cast<cudaEvent_t const*>(events_host), reinterpret_cast<cudaEvent_t const*>(events_host) + n_events);
  return NER_OK;
}

static int train_bwd_impl(const ner_bert_config* cfg, const float* emb_ln_gamma,
                          const ner_bert_layer_weights* layers, const ner_bert_layer_grads* grads,
                          float* d_word_emb, float* d_type_emb, float* d_pos_emb, float* d_emb_ln_gamma,
                          float* d_emb_ln_beta, const int32_t* ids, const int32_t* mask,
                          const int32_t* seg, int B, int L, const int32_t* cu_seqlens, const int32_t* tok_src, int n_packed,
                          float hidden_keep, float attn_keep,
                          uint64_t seed, const float* d_out, const void* saved, size_t saved_bytes,
                          void* scratch, size_t scratch_bytes, ner_stream_t stream) {
  const bool packed = cu_seqlens != nullptr;
  if (!cfg || !layers || !grads || !d_out || !saved || !scratch || !ids || (!mask && !packed) || !emb_ln_gamma) return NER_ERR_INVALID_ARG;
  if (!d_word_emb || !d_type_emb || !d_pos_emb || !d_emb_ln_gamma || !d_emb_ln_beta) return NER_ERR_INVALID_ARG;
  if (B < 0 || L < 1) return NER_ERR_INVALID_ARG;
  if (packed && (!tok_src || n_packed < 0 || n_packed > B * L)) return NER_ERR_INVALID_ARG;
  if (B == 0 || (packed && n_packed == 0)) return NER_OK;
  const int rows = packed ? n_packed : B * L, H = cfg->hidden_size, NH = cfg->num_heads, I = cfg->intermediate_size;
  if (packed) {
    if (saved_bytes < ner_bert_train_packed_saved_bytes(cfg, rows) ||
        scratch_bytes < ner_bert_train_packed_scratch_bytes(cfg, rows, B * L))
      return NER_ERR_WORKSPACE;
  } else
  if (saved_bytes < ner_bert_train_saved_bytes(cfg, rows) || scratch_bytes < ner_bert_train_scratch_bytes(cfg, rows))
    return NER_ERR_WORKSPACE;
  const size_t R = (size_t)rows, lb = layer_saved_bytes(R, H, I);
  const int Rp = (rows + 7) / 8 * 8;
  const size_t W = (size_t)(I > 3 * H ? I : 3 * H);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* base = const_cast<uint8_t*>(static_cast<const uint8_t*>(saved));
  const float* emb_sum = reinterpret_cast<const float*>(base + (size_t)cfg->num_layers * lb);

  uint8_t* p = static_cast<uint8_t*>(scratch);
  float* dA = reinterpret_cast<float*>(p);     p += al(R * H * 4);
  float* dB = reinterpret_cast<float*>(p);     p += al(R * H * 4);
  float* dz32 = reinterpret_cast<float*>(p);   p += al(R * H * 4);
  void* dz16 = p;                              p += al(R * H * 2);
  void* dz16b = p;                             p += al(R * H * 2);
  void* dinter = p;                            p += al(R * I * 2);
  void* dpre = p;                              p += al(R * I * 2);
  void* dctx = p;                              p += al(R * H * 2);
  void* dqkv = p;                              p += al(R * 3 * H * 2);
  void* xt = p;                                p += al(W * Rp * 2);
  void* dyt = p;                               p += al(W * Rp * 2);
  float* dbqkv = reinterpret_cast<float*>(p);  p += al((size_t)3 * H * 4);
  float* dwqkv = reinterpret_cast<float*>(p);  p += al((size_t)3 * H * H * 4);
  float* dpad = reinterpret_cast<float*>(p);   // packed mode: padded [B*L, H] embedding gradient
  const int gelu_erf = cfg->gelu_erf ? 1 : 0;
  const float scale = 1.0f / sqrtf((float)(H / NH));

  const float* d = d_out;   // gradient w.r.t. the current layer's output (f32 [rows, H])
  if (packed) {             // the caller's d_out is padded: keep the real tokens' rows
    NER_TRY(ner_gather_rows(d_out, tok_src, dA, rows, H * 4, stream));
    d = dA;
  }
  for (int l = cfg->num_layers - 1; l >= 0; --l) {
    const ner_bert_layer_weights& w = layers[l];
    const ner_bert_layer_grads& g = grads[l];
    LayerSaved s = carve(base + (size_t)l * lb, R, H, I);
    const uint64_t sa = seed + 1 + 3 * (uint64_t)l, s1 = sa + 1, s2 = sa + 2;
    // The layer's six weight gradients go out as ONE grouped launch at the end of the layer (ner_wgrad_group_bf16: token-major
    // operands read in place, 216 tiles instead of 18..72 per GEMM); shapes the grouped kernel does not take fall back to
    // transposes + one GEMM per gradient.
    const bool grouped = (H % 128 == 0) && (I % 256 == 0) && (H % 256 == 0) && (I % 128 == 0);
    // ---- output LayerNorm + FFN
    NER_TRY(ner_layernorm_dropout_bwd_bias(s.y2, 1, s.x1_32, w.ln2_gamma, d, dz32, dz16, g.d_ln2_gamma, g.d_ln2_beta, g.d_bd, rows,
                                           H, cfg->ln_eps, hidden_keep, s2, stream));   // mask: dense branch (dz16, d_bd) only
    if (!grouped) NER_TRY(wgrad(s.inter, I, nullptr, dz16, H, g.d_wd, rows, Rp, xt, dyt, st));
    NER_TRY(ner_gemm_bf16(dz16, g.wd_kn, nullptr, nullptr, dinter, rows, I, H, NER_EPI_BF16, 0, stream));
    NER_TRY(ner_gelu_bwd_bias_bf16(s.pre, dinter, dpre, g.d_bi, rows, I, gelu_erf, stream));   // d_pre and the FFN1 bias gradient
    if (!grouped) NER_TRY(wgrad(s.x1_16, H, nullptr, dpre, I, g.d_wi, rows, Rp, xt, dyt, st));
    float* dx1 = (d == dA) ? dB : dA;
    NER_TRY(ner_gemm_bf16(dpre, g.wi_kn, nullptr, dz32, dx1, rows, H, I, NER_EPI_RES_F32, 0, stream));
    // ---- attention LayerNorm + output projection
    NER_TRY(ner_layernorm_dropout_bwd_bias(s.y1, 1, s.x32, w.ln1_gamma, dx1, dz32, dz16b, g.d_ln1_gamma, g.d_ln1_beta, g.d_bo, rows,
                                           H, cfg->ln_eps, hidden_keep, s1, stream));
    if (!grouped) NER_TRY(wgrad(s.ctx, H, nullptr, dz16b, H, g.d_wo, rows, Rp, xt, dyt, st));
    NER_TRY(ner_gemm_bf16(dz16b, g.wo_kn, nullptr, nullptr, dctx, rows, H, H, NER_EPI_BF16, 0, stream));
    // ---- attention core + fused QKV projection
    if (packed)
      NER_TRY(ner_bert_attention_bwd_packed(s.qkv, cu_seqlens, s.ctx, dctx, dqkv, B, L, NH, H / NH, scale, attn_keep, sa, stream));
    else
      NER_TRY(ner_bert_attention_bwd(s.qkv, mask, s.ctx, dctx, dqkv, B, L, NH, H / NH, scale, -10000.0f, attn_keep, sa, stream));
    if (cudaMemsetAsync(dbqkv, 0, (size_t)3 * H * 4, st) != cudaSuccess) return NER_ERR_CUDA_BASE - (int)cudaGetLastError();
    NER_TRY(ner_colsum_bf16_add(dqkv, dbqkv, rows, 3 * H, stream));
    NER_TRY(ner_axpy_f32(g.d_bq, dbqkv, H, 1.f, stream));
    NER_TRY(ner_axpy_f32(g.d_bk, dbqkv + H, H, 1.f, stream));
    NER_TRY(ner_axpy_f32(g.d_bv, dbqkv + 2 * H, H, 1.f, stream));
    if (grouped) {
      const ner_wgrad_problem probs[6] = {
          {s.x16, H, dqkv, 3 * H, 0, g.d_wq, H, H},     {s.x16, H, dqkv, 3 * H, H, g.d_wk, H, H},
          {s.x16, H, dqkv, 3 * H, 2 * H, g.d_wv, H, H}, {s.ctx, H, dz16b, H, 0, g.d_wo, H, H},
          {s.x1_16, H, dpre, I, 0, g.d_wi, H, I},       {s.inter, I, dz16, H, 0, g.d_wd, I, H}};
      NER_TRY(ner_wgrad_group_bf16(probs, 6, rows, stream));
    } else {
      // dW_q | dW_k | dW_v: the transposed d_qkv [3H, Rp] is three contiguous [H, Rp] operands
      NER_TRY(ner_transpose_bf16(s.x16, xt, rows, H, Rp, stream));
      NER_TRY(ner_transpose_bf16(dqkv, dyt, rows, 3 * H, Rp, stream));
      NER_TRY(ner_gemm_bf16(xt, dyt, nullptr, nullptr, dwqkv, H, 3 * H, Rp, NER_EPI_F32, 0, stream));
      add_split3_kernel<<<ner_num_sms() * 4, 256, 0, st>>>(dwqkv, g.d_wq, g.d_wk, g.d_wv, H);
      NER_TRY(ner_launch_status());
    }
    float* dprev = (dx1 == dA) ? dB : dA;
    NER_TRY(ner_gemm_bf16(dqkv, g.wqkv_kn, nullptr, dz32, dprev, rows, H, 3 * H, NER_EPI_RES_F32, 0, stream));
    d = dprev;
    if (l < (int)tl_layer_events.size() && tl_layer_events[l] != nullptr &&
        cudaEventRecord(tl_layer_events[l], st) != cudaSuccess)
      return NER_ERR_CUDA_BASE - (int)cudaGetLastError();
  }
  // ---- embeddings: dropout, LayerNorm of (word + type + position), scatter-add
  float* de = (d == dA) ? dB : dA;
  if (hidden_keep < 1.f) {
    NER_TRY(ner_dropout(d, de, R * H, hidden_keep, seed, stream));
    d = de;
  }
  NER_TRY(ner_layernorm_bwd(emb_sum, 0, nullptr, emb_ln_gamma, d, dz32, nullptr, d_emb_ln_gamma, d_emb_ln_beta, rows, H,
                            cfg->ln_eps, stream));
  const float* demb = dz32;
  if (packed) {
    if (cudaMemsetAsync(dpad, 0, (size_t)B * L * H * 4, st) != cudaSuccess) return NER_ERR_CUDA_BASE - (int)cudaGetLastError();
    NER_TRY(ner_scatter_rows(dz32, tok_src, dpad, rows, H * 4, stream));
    demb = dpad;
  }
  return ner_bert_embed_bwd(demb, ids, seg, d_word_emb, d_type_emb, d_pos_emb, B, L, H, cfg->vocab_size, cfg->type_vocab_size,
                            stream);
}

extern "C" int ner_bert_encoder_train_bwd(const ner_bert_config* cfg, const float* emb_ln_gamma,
                                          const ner_bert_layer_weights* layers, const ner_bert_layer_grads* grads,
                                          float* d_word_emb, float* d_type_emb, float* d_pos_emb, float* d_emb_ln_gamma,
                                          float* d_emb_ln_beta, const int32_t* ids, const int32_t* mask,
                                          const int32_t* seg, int B, int L, float hidden_keep, float attn_keep,
                                          uint64_t seed, const float* d_out, const void* saved, size_t saved_bytes,
                                          void* scratch, size_t scratch_bytes, ner_stream_t stream) {
  if (!mask) return NER_ERR_INVALID_ARG;
  return train_bwd_impl(cfg, emb_ln_gamma, layers, grads, d_word_emb, d_type_emb, d_pos_emb, d_emb_ln_gamma, d_emb_ln_beta, ids,
                        mask, seg, B, L, nullptr, nullptr, 0, hidden_keep, attn_keep, seed, d_out, saved, saved_bytes, scratch,
                        scratch_bytes, stream);
}

extern "C" int ner_bert_encoder_train_bwd_packed(const ner_bert_config* cfg, const float* emb_ln_gamma,
                                                 const ner_bert_layer_weights* layers, const ner_bert_layer_grads* grads,
                                                 float* d_word_emb, float* d_type_emb, float* d_pos_emb,
                                                 float* d_emb_ln_gamma, float* d_emb_ln_beta, const int32_t* ids,
                                                 const int32_t* seg, int B, int L, const int32_t* cu_seqlens,
                                                 const int32_t* tok_src, int n_packed, float hidden_keep, float attn_keep,
                                                 uint64_t seed, const float* d_out, const void* saved, size_t saved_bytes,
                                                 void* scratch, size_t scratch_bytes, ner_stream_t stream) {
  if (!cu_seqlens) return NER_ERR_INVALID_ARG;
  return train_bwd_impl(cfg, emb_ln_gamma, layers, grads, d_word_emb, d_type_emb, d_pos_emb, d_emb_ln_gamma, d_emb_ln_beta, ids,
                        nullptr, seg, B, L, cu_seqlens, tok_src, n_packed, hidden_keep, attn_keep, seed, d_out, saved,
                        saved_bytes, scratch, scratch_bytes, stream);
}
