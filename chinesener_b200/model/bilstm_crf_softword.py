# -*-coding:utf-8 -*-
"""`bilstm_crf_softword`: [W[softword_ids] | frozen character embedding] -> bilstm_crf's graph (dropout ->
BiLSTM(128, tanh) -> dropout -> label projection -> CRF).  softword_ids is each character's B/M/E/S word-segmentation
label (data/word_enhance.py SoftWordProc: 0 = none/[PAD], B = 1, M = 2, E = 3, S = 4); W is the trainable [5, 5]
`word_enhance/softword_embedding`, identity at initialisation, whose gradient is ner_small_table_grad's.

The reference's model/bilstm_crf_softword.py and data/word_enhance.py are not in this repository: the graph is restated
from Ma et al., "Simplify the Usage of Lexicon in Chinese NER" (ACL 2020, Softword).  The table's shape, initialisation
and variable name, the label-to-id map and the dropout placement are not pinned to the reference."""
from . import _blocks as nn
from .bilstm_crf import TRAIN_PARAMS as _BILSTM_CRF_PARAMS


def build_graph(features, labels, params, is_training):
    embedding = nn.segmentation_embedding(features, params, is_training, ids=features['softword_ids'])
    return nn.bilstm_crf_tail(embedding, features, params, is_training)


TRAIN_PARAMS = dict(_BILSTM_CRF_PARAMS)
