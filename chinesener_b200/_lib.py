"""ctypes binding of libner_b200.so (the C-ABI in include/ner_b200.h).

The library is the product path: if it is missing or cannot be loaded this module raises —
there is no CPU or PyTorch fallback.  Tensors are passed as raw device pointers; torch is only
the allocator / stream container.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libner_b200.so")

_c = ctypes
_vp, _i = _c.c_void_p, _c.c_int

# name -> (restype, argtypes); must list every symbol include/ner_b200.h declares.
SIGNATURES = {
    "ner_strerror": (_c.c_char_p, [_i]),
    "ner_abi_version": (_i, []),
    "ner_build_info": (_c.c_char_p, []),
    "ner_crf_viterbi": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "ner_crf_viterbi_plan": (_i, [_i, _i, _i, _i, _i]),
    "ner_crf_loglik_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ner_crf_loglik_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c.c_float, _vp, _vp, _i, _i, _i, _vp]),
    "ner_crf_partial_loglik_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ner_crf_partial_loglik_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c.c_float, _vp, _vp, _i, _i, _i, _vp]),
    "ner_crf_distill_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _c.c_float, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ner_crf_distill_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _c.c_float, _vp, _vp, _vp, _c.c_float, _vp, _vp, _vp, _i, _i,
                                 _i, _i, _vp]),
    "ner_crf_viterbi_nbest_workspace_bytes": (_c.c_size_t, [_i, _i, _i, _i]),
    "ner_crf_viterbi_nbest": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _c.c_size_t, _i, _i, _i, _vp]),
    "ner_crf_wide_viterbi_workspace_bytes": (_c.c_size_t, [_i, _i, _i]),
    "ner_crf_wide_viterbi": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _c.c_size_t, _i, _i, _i, _vp]),
    "ner_crf_wide_loglik_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ner_crf_wide_loglik_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c.c_float, _vp, _vp, _i, _i, _i, _vp]),
    "ner_crf_wide_plan": (_i, [_i, _i, _i, _i]),
    "ner_gemm_bf16": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "ner_pack_weight_bf16": (_i, [_vp, _vp, _i, _i, _vp]),
    "ner_cast_bf16": (_i, [_vp, _vp, _c.c_size_t, _vp]),
    "ner_dense_small_n": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "ner_seq_pack_plan": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "ner_bert_embed_ln": (_i, [_vp] * 9 + [_i] * 6 + [_c.c_float, _vp, _i, _vp]),
    "ner_layernorm": (_i, [_vp, _i] + [_vp] * 5 + [_i, _i, _c.c_float, _vp]),
    "ner_layernorm_dropout": (_i, [_vp, _i] + [_vp] * 5 + [_i, _i, _c.c_float, _c.c_float, _c.c_uint64, _vp]),
    "ner_bert_attention": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _c.c_float, _c.c_float, _vp, _i, _c.c_float, _c.c_uint64, _vp]),
    "ner_bilstm_recurrence": (_i, [_vp] * 5 + [_i, _i, _i, _i, _c.c_float, _vp, _vp, _vp, _vp, _c.c_float, _c.c_uint64, _vp]),
    "ner_bilstm_recurrence_bwd": (_i, [_vp] * 7 + [_i, _i, _i, _i, _c.c_float, _c.c_uint64, _vp]),
    "ner_bigru_recurrence": (_i, [_vp] * 5 + [_i, _i, _i, _i, _i] + [_vp] * 4 + [_c.c_float, _c.c_uint64, _vp]),
    "ner_bigru_recurrence_bwd": (_i, [_vp] * 7 + [_i, _i, _i, _i, _c.c_float, _c.c_uint64, _vp]),
    "ner_rnn_plan": (_i, [_i] * 5 + [_c.POINTER(_i)] * 3),
    "ner_transpose_cast_bf16": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "ner_colsum_add": (_i, [_vp, _vp, _i, _i, _i, _c.c_float, _vp]),
    "ner_dense_small_n_bwd": (_i, [_vp] * 6 + [_i, _i, _i, _vp]),
    "ner_dropout": (_i, [_vp, _vp, _c.c_size_t, _c.c_float, _c.c_uint64, _vp]),
    "ner_relu_bwd_f32": (_i, [_vp, _vp, _vp, _c.c_size_t, _vp]),
    "ner_relu_f32": (_i, [_vp, _vp, _c.c_size_t, _vp]),
    "ner_reduce_max_time": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "ner_reduce_max_time_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _c.c_float, _vp]),
    "ner_softmax_xent": (_i, [_vp, _vp, _vp, _vp, _i, _i, _c.c_float, _vp]),
    "ner_attention_f32_bwd": (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _c.c_float, _vp, _i, _vp, _i, _vp, _i, _vp, _i,
                                   _vp, _vp, _i, _i, _i, _i, _vp]),
    "ner_dropout_bf16": (_i, [_vp, _vp, _c.c_size_t, _c.c_float, _c.c_uint64, _vp]),
    "ner_sumsq_add": (_i, [_vp, _c.c_size_t, _vp, _vp, _vp]),
    "ner_sumsq_scratch_floats": (_c.c_size_t, []),
    "ner_token_xent": (_i, [_vp] * 6 + [_c.c_float, _vp, _i, _i, _i, _vp]),
    "ner_token_xent_scratch_floats": (_c.c_size_t, []),
    "ner_token_dice": (_i, [_vp] * 6 + [_c.c_float] * 3 + [_vp, _i, _i, _i, _vp]),
    "ner_mlm_mask": (_i, [_vp] * 4 + [_i, _i, _c.c_uint64, _i, _i] + [_vp] * 4),
    "ner_vocab_xent_scratch_floats": (_c.c_size_t, [_i]),
    "ner_vocab_xent": (_i, [_vp, _i, _vp, _i, _i, _c.c_float] + [_vp] * 7),
    "ner_augment_rows_smem_bytes": (_c.c_size_t, [_i]),
    "ner_augment_rows": (_i, [_vp] * 5 + [_i, _i, _vp, _i, _vp, _i] + [_vp] * 3 + [_i, _i, _vp, _vp, _i]
                         + [_c.c_float] * 5 + [_c.c_uint64, _i, _i, _i] + [_vp] * 7 + [_vp]),
    "ner_vocab_sample": (_i, [_vp, _i, _i, _vp, _vp, _i, _c.c_longlong, _c.c_float, _c.c_uint64, _vp, _vp]),
    "ner_mrc_pairs": (_i, [_vp] * 6 + [_i] * 6 + [_vp] * 7),
    "ner_mrc_merge": (_i, [_vp] * 3 + [_i] * 6 + [_vp, _vp]),
    "ner_mrc_span_targets": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "ner_mrc_span_match_fwd_workspace_bytes": (_c.c_size_t, [_i, _i]),
    "ner_mrc_span_match_fwd": (_i, [_vp, _i] + [_vp] * 5 + [_i] * 3 + [_c.c_float, _c.c_uint64] + [_vp] * 3
                               + [_c.c_size_t, _vp]),
    "ner_mrc_span_match_bwd_workspace_bytes": (_c.c_size_t, [_i, _i]),
    "ner_mrc_span_match_bwd": (_i, [_vp, _i] + [_vp] * 5 + [_i] * 3 + [_c.c_float, _c.c_float, _c.c_uint64] + [_vp] * 5
                               + [_c.c_size_t, _vp]),
    "ner_mrc_span_decode_workspace_bytes": (_c.c_size_t, [_i, _i]),
    "ner_mrc_span_decode": (_i, [_vp] * 3 + [_i] + [_vp] * 5 + [_i] * 8 + [_vp] * 5 + [_c.c_size_t, _vp]),
    "ner_gp_targets": (_i, [_vp] * 3 + [_i] * 3 + [_vp, _vp]),
    "ner_gp_rope": (_i, [_vp, _i, _vp] + [_i] * 3 + [_vp] * 3),
    "ner_gp_rope_bwd": (_i, [_vp, _vp] + [_i] * 3 + [_vp, _i, _vp]),
    "ner_gp_loss_workspace_bytes": (_c.c_size_t, [_i] * 3),
    "ner_gp_loss_fwd": (_i, [_vp] * 5 + [_i] * 3 + [_vp] * 3 + [_c.c_size_t, _vp]),
    "ner_gp_loss_bwd": (_i, [_vp] * 5 + [_i] * 3 + [_c.c_float, _vp, _vp]),
    "ner_gp_decode_workspace_bytes": (_c.c_size_t, [_i] * 3),
    "ner_gp_decode": (_i, [_vp] * 5 + [_i] * 7 + [_vp] * 5 + [_c.c_size_t, _vp]),
    "ner_window_plan": (_i, [_vp] * 3 + [_i] * 5 + [_vp] * 6),
    "ner_layernorm_bwd": (_i, [_vp, _i] + [_vp] * 7 + [_i, _i, _c.c_float, _vp]),
    "ner_layernorm_dropout_bwd": (_i, [_vp, _i] + [_vp] * 7 + [_i, _i, _c.c_float, _c.c_float, _c.c_uint64, _vp]),
    "ner_layernorm_dropout_bwd_bias": (_i, [_vp, _i] + [_vp] * 8 + [_i, _i, _c.c_float, _c.c_float, _c.c_uint64, _vp]),
    "ner_transpose_bf16": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "ner_colsum_bf16_add": (_i, [_vp, _vp, _i, _i, _vp]),
    "ner_gelu_bf16": (_i, [_vp, _vp, _c.c_size_t, _i, _vp]),
    "ner_gelu_f32": (_i, [_vp, _vp, _c.c_size_t, _i, _vp]),
    "ner_gelu_bwd_bf16": (_i, [_vp, _vp, _vp, _c.c_size_t, _i, _vp]),
    "ner_gelu_bwd_bias_bf16": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "ner_bert_embed_bwd": (_i, [_vp] * 6 + [_i] * 5 + [_vp]),
    "ner_bert_attention_bwd": (_i, [_vp] * 5 + [_i] * 4 + [_c.c_float, _c.c_float, _c.c_float, _c.c_uint64, _vp]),
    "ner_bert_attention_bwd_packed": (_i, [_vp] * 5 + [_i] * 4 + [_c.c_float, _c.c_float, _c.c_uint64, _vp]),
    "ner_gather_rows": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "ner_scatter_rows": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "ner_adam_step": (_i, [_vp] * 4 + [_c.c_size_t] + [_c.c_float] * 5 + [_i, _c.c_float, _vp, _c.c_float, _vp]),
    "ner_softlexicon_pool_fwd": (_i, [_vp] * 4 + [_i] * 6 + [_vp]),
    "ner_embedding_lookup": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ner_cast_pad_bf16": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "ner_split_bf16": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ner_attention_f32": (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _c.c_float, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ner_softlexicon_pool_bwd": (_i, [_vp] * 4 + [_i] * 5 + [_vp]),
    "ner_multihot_embed_fwd": (_i, [_vp] * 3 + [_i] * 4 + [_vp]),
    "ner_small_table_grad_scratch_floats": (_c.c_size_t, [_i, _i]),
    "ner_small_table_grad": (_i, [_vp] * 4 + [_i] * 4 + [_vp, _vp]),
    "ner_gemm_e4m3": (_i, [_vp] * 7 + [_i] * 4 + [_vp]),
    "ner_quantize_weight_e4m3": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "ner_bert_embed_ln_e4m3": (_i, [_vp] * 11 + [_i] * 6 + [_c.c_float, _vp, _i, _vp]),
    "ner_layernorm_e4m3": (_i, [_vp, _i] + [_vp] * 7 + [_i, _i, _c.c_float, _vp]),
}



class BertConfig(_c.Structure):
    _fields_ = [("hidden_size", _i), ("num_heads", _i), ("intermediate_size", _i), ("num_layers", _i),
                ("vocab_size", _i), ("type_vocab_size", _i), ("max_position", _i), ("ln_eps", _c.c_float),
                ("gelu_erf", _i), ("gemm_tile", _i)]


class BertLayerWeights(_c.Structure):
    _fields_ = [(n, _vp) for n in ("wqkv", "bqkv", "wo", "bo", "ln1_gamma", "ln1_beta", "wi", "bi", "wd", "bd",
                                   "ln2_gamma", "ln2_beta")]


class BertLayerWeightsFp8(_c.Structure):
    _fields_ = [(n, _vp) for n in ("wqkv", "sqkv", "bqkv", "wo", "bo", "ln1_gamma", "ln1_beta", "wi", "si", "bi", "wd", "sd",
                                   "bd", "ln2_gamma", "ln2_beta")]


class BertLayerGrads(_c.Structure):
    _fields_ = [(n, _vp) for n in ("wqkv_kn", "wo_kn", "wi_kn", "wd_kn", "d_wq", "d_wk", "d_wv", "d_bq", "d_bk", "d_bv",
                                   "d_wo", "d_bo", "d_ln1_gamma", "d_ln1_beta", "d_wi", "d_bi", "d_wd", "d_bd",
                                   "d_ln2_gamma", "d_ln2_beta")]


SIGNATURES["ner_bert_train_saved_bytes"] = (_c.c_size_t, [_c.POINTER(BertConfig), _i])
SIGNATURES["ner_bert_train_scratch_bytes"] = (_c.c_size_t, [_c.POINTER(BertConfig), _i])
SIGNATURES["ner_bert_encoder_train_fwd"] = (_i, [_c.POINTER(BertConfig)] + [_vp] * 5 + [_c.POINTER(BertLayerWeights)] + [_vp] * 3
                                            + [_i, _i, _c.c_float, _c.c_float, _c.c_uint64, _vp, _vp, _vp, _c.c_size_t, _vp])
SIGNATURES["ner_bert_encoder_train_bwd"] = (_i, [_c.POINTER(BertConfig), _vp, _c.POINTER(BertLayerWeights), _c.POINTER(BertLayerGrads)]
                                            + [_vp] * 5 + [_vp] * 3 + [_i, _i, _c.c_float, _c.c_float, _c.c_uint64, _vp, _vp,
                                                                       _c.c_size_t, _vp, _c.c_size_t, _vp])
SIGNATURES["ner_bert_train_packed_saved_bytes"] = (_c.c_size_t, [_c.POINTER(BertConfig), _i])
SIGNATURES["ner_bert_train_packed_scratch_bytes"] = (_c.c_size_t, [_c.POINTER(BertConfig), _i, _i])
SIGNATURES["ner_bert_encoder_train_fwd_packed"] = (_i, [_c.POINTER(BertConfig)] + [_vp] * 5 + [_c.POINTER(BertLayerWeights)] + [_vp] * 2
                                                   + [_i, _i, _vp, _vp, _i, _c.c_float, _c.c_float, _c.c_uint64, _vp, _vp, _vp,
                                                      _c.c_size_t, _vp])
SIGNATURES["ner_bert_encoder_train_bwd_packed"] = (_i, [_c.POINTER(BertConfig), _vp, _c.POINTER(BertLayerWeights),
                                                        _c.POINTER(BertLayerGrads)] + [_vp] * 5 + [_vp] * 2
                                                   + [_i, _i, _vp, _vp, _i, _c.c_float, _c.c_float, _c.c_uint64, _vp, _vp,
                                                      _c.c_size_t, _vp, _c.c_size_t, _vp])
SIGNATURES["ner_bert_bilstm_crf_predict_workspace_bytes"] = (_c.c_size_t, [_c.POINTER(BertConfig), _i, _i, _i, _i, _i])
SIGNATURES["ner_bert_bilstm_crf_predict"] = (_i, [_c.POINTER(BertConfig)] + [_vp] * 5 + [_c.POINTER(BertLayerWeights)] + [_vp] * 4
                                             + [_i, _i] + [_vp] * 3 + [_i] + [_vp] * 4 + [_i, _i, _i, _vp, _vp, _c.c_size_t, _vp])
SIGNATURES["ner_bert_embed_sum"] = (_i, [_vp] * 6 + [_i] * 6 + [_vp])
SIGNATURES["ner_axpy_f32"] = (_i, [_vp, _vp, _c.c_size_t, _c.c_float, _vp])
SIGNATURES["ner_bert_encoder_workspace_bytes"] = (_c.c_size_t, [_c.POINTER(BertConfig), _i])
SIGNATURES["ner_bert_encoder_fwd"] = (_i, [_c.POINTER(BertConfig)] + [_vp] * 5 + [_c.POINTER(BertLayerWeights)] + [_vp] * 3
                                      + [_i, _i, _vp, _vp, _i, _vp, _vp, _vp, _c.c_size_t, _vp])
SIGNATURES["ner_bert_encoder_fp8_workspace_bytes"] = (_c.c_size_t, [_c.POINTER(BertConfig), _i])
SIGNATURES["ner_bert_encoder_fwd_fp8"] = (_i, [_c.POINTER(BertConfig)] + [_vp] * 5 + [_c.POINTER(BertLayerWeightsFp8)] + [_vp] * 3
                                          + [_i, _i, _vp, _vp, _i, _vp, _vp, _vp, _c.c_size_t, _vp])

class PackEntry(_c.Structure):
    _fields_ = [("src", _vp), ("K", _i), ("N", _i), ("dst_nk_bf16", _vp), ("ld_nk", _i), ("dst_kn_bf16", _vp), ("ld_kn", _i)]


SIGNATURES["ner_pack_weights_group_bf16"] = (_i, [_vp, _vp, _i, _i, _vp])


class WgradProblem(_c.Structure):
    _fields_ = [("x_bf16", _vp), ("ld_x", _i), ("dy_bf16", _vp), ("ld_dy", _i), ("dy_col0", _i), ("dw", _vp), ("k_in", _i),
                ("n_out", _i)]


SIGNATURES["ner_wgrad_group_bf16"] = (_i, [_c.POINTER(WgradProblem), _i, _i, _vp])
SIGNATURES["ner_bert_train_bwd_set_layer_events"] = (_i, [_vp, _i])
SIGNATURES["ner_extract_spans"] = (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp])
SIGNATURES["ner_extract_spans_wide"] = (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp])
SIGNATURES["ner_featurize_wordpiece"] = (_i, [_vp] * 3 + [_i, _i] + [_vp] * 4 + [_i, _vp, _vp] + [_i] * 6 + [_vp] * 6)
SIGNATURES["ner_featurize_chars"] = (_i, [_vp] * 3 + [_i, _i] + [_vp] * 3 + [_i, _vp, _vp, _i, _i] + [_vp] * 6)
SIGNATURES["ner_lexicon_create"] = (_vp, [_vp, _vp, _vp, _i])
SIGNATURES["ner_lexicon_destroy"] = (None, [_vp])
SIGNATURES["ner_lexicon_num_nodes"] = (_c.c_int64, [_vp])
SIGNATURES["ner_lexicon_build"] = (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _i, _vp, _vp, _i])
SIGNATURES["ner_lexicon_build_lattice"] = (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _i])
SIGNATURES["ner_lattice_recurrence"] = (_i, [_vp] * 9 + [_i] * 4 + [_vp] * 8)
SIGNATURES["ner_lattice_recurrence_bwd"] = (_i, [_vp] * 16 + [_i] * 4 + [_vp])

# return values of ner_crf_viterbi_plan, by enum value (include/ner_b200.h: NER_VIT_*)
VIT_PLANS = ("small", "tma", "parked", "onchip_128", "onchip_32", "small_any_b", "none")

_lib = None


class NerB200Error(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle; raises if the extension is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NerB200Error(
                f"{LIB_PATH} not found: build it with `python -m chinesener_b200.build` "
                "(there is no CPU fallback for the sm_90a kernels)")
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


LAUNCHES = 0     # kernel launches issued through the C-ABI (every successful call launches one kernel)
_HOOK = None     # optional profiling hook: fn(name) -> context manager, set by bench.py


def check(status):
    global LAUNCHES
    LAUNCHES += 1
    if status != 0:
        raise NerB200Error(lib().ner_strerror(status).decode())


def ptr(t):
    return 0 if t is None else t.data_ptr()


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def stream():
    """cudaStream_t of torch's current stream.  The raw getter avoids building a torch.cuda.Stream object per
    call: with a non-default stream current (predict_iter(streams>1)) that wrapper costs more host time per call
    than the launches it wraps."""
    if _raw_stream is not None:
        return _raw_stream(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise NerB200Error("ner_b200 kernels take CUDA tensors (got a CPU tensor); there is no CPU path")
        if t is not None and not t.is_contiguous():
            raise NerB200Error("ner_b200 kernels take contiguous row-major tensors")
