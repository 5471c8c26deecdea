// One C-ABI call for the whole PREDICT step of the bert_bilstm_crf plugin (reference
// model/bert_bilstm_crf.py:8-34 in PREDICT mode: pretrain_bert_embedding -> bilstm -> dense(logits) ->
// crf_decode; the log-likelihood of crf_layer is not fetched by PREDICT, tools/train_utils.py:181-185).
// The host enqueues: packing plan, packed BERT encoder, LSTM input projection (wgmma GEMM), the
// bidirectional recurrence, the label projection and Viterbi — the same kernels the layer functions of
// chinesener_b200/tools/layer.py launch one by one, in the same order, on the caller's stream.  It exists to
// take the ~20 Python-level calls of a step off the host's critical path when eight 4-stream pipelines share
// one host (DESIGN.md §7); build_graph() stays the definition and tests/test_models_gpu.py pins the equality.
#include "common.cuh"

namespace {
inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }
}  // namespace

extern "C" size_t ner_bert_bilstm_crf_predict_workspace_bytes(const ner_bert_config* cfg, int B, int L, int rows,
                                                              int lstm_hidden, int num_tags) {
  if (!cfg || B < 0 || L < 1 || rows < 0) return 0;
  const size_t H = (size_t)cfg->hidden_size, R = (size_t)rows, Hl = (size_t)lstm_hidden;
  return al256((size_t)(B + 1) * 4)            // cu_seqlens
         + al256((size_t)B * L * 4)            // tok_src
         + al256(R * H * 4) + al256(R * H * 2)  // sequence_output f32 / bf16 (packed rows)
         + al256(R * 8 * Hl * 4)               // LSTM input projection
         + al256((size_t)B * L * 2 * Hl * 4)   // BiLSTM output
         + al256((size_t)B * L * num_tags * 4)  // emission logits
         + ner_bert_encoder_workspace_bytes(cfg, rows);
}

extern "C" int ner_bert_bilstm_crf_predict(const ner_bert_config* cfg, const float* word_emb, const float* type_emb,
                                           const float* pos_emb, const float* emb_ln_gamma, const float* emb_ln_beta,
                                           const ner_bert_layer_weights* layers, const void* lstm_wx_bf16,
                                           const float* lstm_bias, const float* lstm_wh_fw, const float* lstm_wh_bw,
                                           int lstm_hidden, int lstm_activation, const float* logits_w,
                                           const float* logits_b, const float* trans, int num_tags, const int32_t* ids,
                                           const int32_t* mask, const int32_t* seg, const int32_t* seq_len, int B, int L,
                                           int n_packed, int32_t* pred_ids, void* workspace, size_t workspace_bytes,
                                           ner_stream_t stream) {
  if (!cfg || !layers || !lstm_wx_bf16 || !lstm_bias || !lstm_wh_fw || !lstm_wh_bw || !logits_w || !logits_b || !trans ||
      !ids || !mask || !seq_len || !pred_ids || !workspace)
    return NER_ERR_INVALID_ARG;
  if (B < 0 || L < 1 || n_packed < 0 || n_packed > B * L) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  const int H = cfg->hidden_size, Hl = lstm_hidden, K = num_tags;
  if (H % 8 != 0) return NER_ERR_UNSUPPORTED;   // the bf16 sequence output is the GEMM A operand as is
  if (workspace_bytes < ner_bert_bilstm_crf_predict_workspace_bytes(cfg, B, L, n_packed, Hl, K)) return NER_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* p = static_cast<uint8_t*>(workspace);
  int32_t* cu = reinterpret_cast<int32_t*>(p);       p += al256((size_t)(B + 1) * 4);
  int32_t* tok_src = reinterpret_cast<int32_t*>(p);  p += al256((size_t)B * L * 4);
  float* x32 = reinterpret_cast<float*>(p);          p += al256((size_t)n_packed * H * 4);
  void* x16 = p;                                     p += al256((size_t)n_packed * H * 2);
  float* xproj = reinterpret_cast<float*>(p);        p += al256((size_t)n_packed * 8 * Hl * 4);
  float* lstm_out = reinterpret_cast<float*>(p);     p += al256((size_t)B * L * 2 * Hl * 4);
  float* logits = reinterpret_cast<float*>(p);       p += al256((size_t)B * L * K * 4);
  void* enc_ws = p;
  const size_t enc_bytes = ner_bert_encoder_workspace_bytes(cfg, n_packed);

  int rc = ner_seq_pack_plan(mask, cu, tok_src, B, L, stream);
  if (rc != NER_OK) return rc;
  if (n_packed == 0) {   // every sentence empty: all-zero tags
    if (cudaMemsetAsync(pred_ids, 0, (size_t)B * L * 4, st) != cudaSuccess) return NER_ERR_CUDA_BASE - (int)cudaGetLastError();
    return NER_OK;
  }
  rc = ner_bert_encoder_fwd(cfg, word_emb, type_emb, pos_emb, emb_ln_gamma, emb_ln_beta, layers, ids, mask, seg, B, L, cu,
                            tok_src, n_packed, x32, x16, enc_ws, enc_bytes, stream);
  if (rc != NER_OK) return rc;
  rc = ner_gemm_bf16(x16, lstm_wx_bf16, lstm_bias, nullptr, xproj, n_packed, 8 * Hl, H, NER_EPI_F32, cfg->gemm_tile, stream);
  if (rc != NER_OK) return rc;
  rc = ner_bilstm_recurrence(xproj, lstm_wh_fw, lstm_wh_bw, seq_len, lstm_out, B, L, Hl, lstm_activation, 1.0f, cu, nullptr,
                             nullptr, nullptr, 1.0f, 0, stream);
  if (rc != NER_OK) return rc;
  rc = ner_dense_small_n(lstm_out, 0, logits_w, logits_b, logits, B * L, 2 * Hl, K, nullptr, stream);
  if (rc != NER_OK) return rc;
  return ner_crf_viterbi(logits, seq_len, trans, pred_ids, nullptr, B, L, K, stream);
}
