// One C-ABI call for the whole BertModel forward (bert_base.bert.modeling.BertModel as driven
// from reference tools/layer.py:63-81): embedding+LN, then per layer
//   fused-QKV GEMM -> attention -> out-proj GEMM(+bias, bf16) -> LayerNorm(+f32 residual)
//   -> FFN1 GEMM(+bias+GELU) -> FFN2 GEMM(+bias, bf16) -> LayerNorm(+f32 residual).
// The residual stream itself stays fp32 (LayerNorm writes an f32 and a bf16 copy); only the
// dense sub-layer outputs are rounded to bf16 before the add.
// The host loop below only enqueues kernels (7 per layer) on the caller's stream; doing it here
// instead of from Python removes ~85 ctypes round trips per step.
#include "common.cuh"

namespace {
inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
}  // namespace

extern "C" size_t ner_bert_encoder_workspace_bytes(const ner_bert_config* cfg, int rows) {
  if (!cfg || rows < 0) return 0;
  const size_t R = (size_t)rows, H = (size_t)cfg->hidden_size, I = (size_t)cfg->intermediate_size;
  return align256(R * 3 * H * 2)    // qkv  bf16
         + align256(R * H * 2)      // ctx  bf16
         + align256(R * H * 4)      // y    bf16 dense output (LayerNorm adds the f32 residual); f32-sized
         + align256(R * H * 4)      // x1   f32 (post-attention LayerNorm)
         + align256(R * H * 2)      // x1   bf16
         + align256(R * I * 2);     // FFN intermediate bf16
}

extern "C" int ner_bert_encoder_fwd(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                                    const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                                    const ner_bert_layer_weights* layers, const int32_t* ids, const int32_t* mask,
                                    const int32_t* seg, int B, int L, const int32_t* cu_seqlens,
                                    const int32_t* tok_src, int n_packed, float* out_f32, void* out_bf16,
                                    void* workspace, size_t workspace_bytes, ner_stream_t stream) {
  if (!cfg || !layers || !out_f32 || !out_bf16) return NER_ERR_INVALID_ARG;
  if (B < 0 || L < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  const bool packed = cu_seqlens != nullptr;
  if (packed != (tok_src != nullptr)) return NER_ERR_INVALID_ARG;
  const int rows = packed ? n_packed : B * L;
  if (rows < 0 || rows > B * L) return NER_ERR_INVALID_ARG;
  if (rows == 0) return NER_OK;
  const int H = cfg->hidden_size, NH = cfg->num_heads, I = cfg->intermediate_size;
  if (H % NH != 0) return NER_ERR_INVALID_ARG;
  if (workspace_bytes < ner_bert_encoder_workspace_bytes(cfg, rows) || !workspace) return NER_ERR_WORKSPACE;

  uint8_t* p = static_cast<uint8_t*>(workspace);
  void* qkv = p;   p += align256((size_t)rows * 3 * H * 2);
  void* ctx = p;   p += align256((size_t)rows * H * 2);
  float* y = reinterpret_cast<float*>(p);    p += align256((size_t)rows * H * 4);
  float* x1f = reinterpret_cast<float*>(p);  p += align256((size_t)rows * H * 4);
  void* x1b = p;   p += align256((size_t)rows * H * 2);
  void* inter = p;

  int rc = ner_bert_embed_ln(word_emb, type_emb, pos_emb, emb_ln_gamma, emb_ln_beta, ids, seg, out_f32, out_bf16, B, L, H,
                             cfg->vocab_size, cfg->type_vocab_size, cfg->max_position, cfg->ln_eps, tok_src, n_packed,
                             stream);
  if (rc != NER_OK) return rc;
  const int gelu = cfg->gelu_erf ? NER_EPI_GELU_ERF_BF16 : NER_EPI_GELU_TANH_BF16;
  const float scale = 1.0f / sqrtf((float)(H / NH));
  for (int l = 0; l < cfg->num_layers; ++l) {
    const ner_bert_layer_weights& w = layers[l];
    rc = ner_gemm_bf16(out_bf16, w.wqkv, w.bqkv, nullptr, qkv, rows, 3 * H, H, NER_EPI_BF16, cfg->gemm_tile, stream);
    if (rc != NER_OK) return rc;
    rc = ner_bert_attention(qkv, mask, ctx, B, L, NH, H / NH, scale, -10000.0f, cu_seqlens, rows, 1.0f, 0, stream);
    if (rc != NER_OK) return rc;
    rc = ner_gemm_bf16(ctx, w.wo, w.bo, nullptr, y, rows, H, H, NER_EPI_BF16, cfg->gemm_tile, stream);
    if (rc != NER_OK) return rc;
    rc = ner_layernorm(y, 1, out_f32, w.ln1_gamma, w.ln1_beta, x1f, x1b, rows, H, cfg->ln_eps, stream);
    if (rc != NER_OK) return rc;
    rc = ner_gemm_bf16(x1b, w.wi, w.bi, nullptr, inter, rows, I, H, gelu, cfg->gemm_tile, stream);
    if (rc != NER_OK) return rc;
    rc = ner_gemm_bf16(inter, w.wd, w.bd, nullptr, y, rows, H, I, NER_EPI_BF16, cfg->gemm_tile, stream);
    if (rc != NER_OK) return rc;
    rc = ner_layernorm(y, 1, x1f, w.ln2_gamma, w.ln2_beta, out_f32, out_bf16, rows, H, cfg->ln_eps, stream);
    if (rc != NER_OK) return rc;
  }
  return NER_OK;
}

// FP8 inference encoder: the same layer with QKV, FFN1 and FFN2 on ner_gemm_e4m3.  Per layer
//   QKV e4m3 GEMM (A = e4m3 copy of the previous LayerNorm) -> attention -> out-proj bf16 GEMM -> LayerNorm (f32 + e4m3)
//   -> FFN1 e4m3 GEMM (+bias, GELU -> e4m3) -> FFN2 e4m3 GEMM (+bias, bf16) -> LayerNorm (f32 + e4m3, or f32 + bf16 after
//   the last layer: sequence_output and its bf16 copy, as ner_bert_encoder_fwd writes them).
extern "C" size_t ner_bert_encoder_fp8_workspace_bytes(const ner_bert_config* cfg, int rows) {
  if (!cfg || rows < 0) return 0;
  const size_t R = (size_t)rows, H = (size_t)cfg->hidden_size, I = (size_t)cfg->intermediate_size;
  return align256(R * 3 * H * 2)      // qkv  bf16
         + align256(R * H * 2)        // ctx  bf16
         + align256(R * H * 2)        // y    bf16 dense output
         + align256(R * H * 4)        // x1   f32 (post-attention LayerNorm)
         + align256(R * H)            // e4m3 LayerNorm output (QKV / FFN1 operand)
         + align256(R * (H / 128) * 4)   //   its block scales
         + align256(R * I)            // FFN intermediate e4m3
         + align256(R * (I / 128) * 4);  //   its block scales
}

extern "C" int ner_bert_encoder_fwd_fp8(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                                        const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                                        const ner_bert_layer_weights_fp8* layers, const int32_t* ids, const int32_t* mask,
                                        const int32_t* seg, int B, int L, const int32_t* cu_seqlens, const int32_t* tok_src,
                                        int n_packed, float* out_f32, void* out_bf16, void* workspace,
                                        size_t workspace_bytes, ner_stream_t stream) {
  if (!cfg || !layers || !out_f32 || !out_bf16) return NER_ERR_INVALID_ARG;
  if (B < 0 || L < 1) return NER_ERR_INVALID_ARG;
  const int H = cfg->hidden_size, NH = cfg->num_heads, I = cfg->intermediate_size;
  if (NH < 1 || H % NH != 0 || cfg->num_layers < 1) return NER_ERR_INVALID_ARG;
  if (H % 128 != 0 || I % 128 != 0) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  const bool packed = cu_seqlens != nullptr;
  if (packed != (tok_src != nullptr)) return NER_ERR_INVALID_ARG;
  const int rows = packed ? n_packed : B * L;
  if (rows < 0 || rows > B * L) return NER_ERR_INVALID_ARG;
  if (rows == 0) return NER_OK;
  if (workspace_bytes < ner_bert_encoder_fp8_workspace_bytes(cfg, rows) || !workspace) return NER_ERR_WORKSPACE;

  uint8_t* p = static_cast<uint8_t*>(workspace);
  void* qkv = p;   p += align256((size_t)rows * 3 * H * 2);
  void* ctx = p;   p += align256((size_t)rows * H * 2);
  void* y = p;     p += align256((size_t)rows * H * 2);
  float* x1f = reinterpret_cast<float*>(p);  p += align256((size_t)rows * H * 4);
  void* xq = p;    p += align256((size_t)rows * H);
  float* xs = reinterpret_cast<float*>(p);   p += align256((size_t)rows * (H / 128) * 4);
  void* iq = p;    p += align256((size_t)rows * I);
  float* is = reinterpret_cast<float*>(p);

  int rc = ner_bert_embed_ln_e4m3(word_emb, type_emb, pos_emb, emb_ln_gamma, emb_ln_beta, ids, seg, out_f32, nullptr, xq, xs,
                                  B, L, H, cfg->vocab_size, cfg->type_vocab_size, cfg->max_position, cfg->ln_eps, tok_src,
                                  n_packed, stream);
  if (rc != NER_OK) return rc;
  const int gelu = cfg->gelu_erf ? NER_EPI_GELU_ERF_E4M3 : NER_EPI_GELU_TANH_E4M3;
  const float scale = 1.0f / sqrtf((float)(H / NH));
  for (int l = 0; l < cfg->num_layers; ++l) {
    const ner_bert_layer_weights_fp8& w = layers[l];
    rc = ner_gemm_e4m3(xq, xs, w.wqkv, w.sqkv, w.bqkv, qkv, nullptr, rows, 3 * H, H, NER_EPI_BF16, stream);
    if (rc != NER_OK) return rc;
    rc = ner_bert_attention(qkv, mask, ctx, B, L, NH, H / NH, scale, -10000.0f, cu_seqlens, rows, 1.0f, 0, stream);
    if (rc != NER_OK) return rc;
    rc = ner_gemm_bf16(ctx, w.wo, w.bo, nullptr, y, rows, H, H, NER_EPI_BF16, cfg->gemm_tile, stream);
    if (rc != NER_OK) return rc;
    rc = ner_layernorm_e4m3(y, 1, out_f32, w.ln1_gamma, w.ln1_beta, x1f, nullptr, xq, xs, rows, H, cfg->ln_eps, stream);
    if (rc != NER_OK) return rc;
    rc = ner_gemm_e4m3(xq, xs, w.wi, w.si, w.bi, iq, is, rows, I, H, gelu, stream);
    if (rc != NER_OK) return rc;
    rc = ner_gemm_e4m3(iq, is, w.wd, w.sd, w.bd, y, nullptr, rows, H, I, NER_EPI_BF16, stream);
    if (rc != NER_OK) return rc;
    if (l + 1 < cfg->num_layers)
      rc = ner_layernorm_e4m3(y, 1, x1f, w.ln2_gamma, w.ln2_beta, out_f32, nullptr, xq, xs, rows, H, cfg->ln_eps, stream);
    else
      rc = ner_layernorm(y, 1, x1f, w.ln2_gamma, w.ln2_beta, out_f32, out_bf16, rows, H, cfg->ln_eps, stream);
    if (rc != NER_OK) return rc;
  }
  return NER_OK;
}
