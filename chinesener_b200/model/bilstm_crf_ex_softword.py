# -*-coding:utf-8 -*-
"""`bilstm_crf_ex_softword`: [ex_softword_ids · W | frozen character embedding] -> bilstm_crf's graph (dropout ->
BiLSTM(128, tanh) -> dropout -> label projection -> CRF).  ex_softword_ids [B, L * 5] is each character's multi-hot
B/M/E/S/None label set from the lexicon match (data/word_enhance.py ExSoftWordProc); W is the trainable [5, 5]
`word_enhance/softword_embedding`, identity at initialisation.  The projection is ner_multihot_embed_fwd, W's gradient
ner_small_table_grad.

The reference's model/bilstm_crf_ex_softword.py and data/word_enhance.py are not in this repository: the graph is
restated from Ma et al., "Simplify the Usage of Lexicon in Chinese NER" (ACL 2020, ExSoftword).  The table's shape,
initialisation and variable name, the label layout and the dropout placement are not pinned to the reference."""
from . import _blocks as nn
from .bilstm_crf import TRAIN_PARAMS as _BILSTM_CRF_PARAMS


def build_graph(features, labels, params, is_training):
    embedding = nn.segmentation_embedding(features, params, is_training, weights=features['ex_softword_ids'])
    return nn.bilstm_crf_tail(embedding, features, params, is_training)


TRAIN_PARAMS = dict(_BILSTM_CRF_PARAMS)
