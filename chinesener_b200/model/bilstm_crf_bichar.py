# -*-coding:utf-8 -*-
"""`bilstm_crf_bichar`: [frozen character embedding | frozen bi-character embedding] -> bilstm_crf's graph (dropout ->
BiLSTM(128, tanh) -> dropout -> label projection -> CRF).

The reference's model/bilstm_crf_bichar.py is not in this repository: the graph is restated from bilstm_crf and the
bigram input of TENER (transformer_tener_crf_bichar), and the dropout placement (embedding_dropout on the concatenated
input, i.e. on each piece) is not pinned to it.  Both tables are constants, so TRAIN records no embedding gradient."""
import torch

from .. import ops
from . import _blocks as nn
from .bilstm_crf import TRAIN_PARAMS as _BILSTM_CRF_PARAMS


def build_graph(features, labels, params, is_training):
    input_ids = features['token_ids']
    B, L = input_ids.shape
    char_table = nn.device_constant(params, 'embedding')
    bichar_table = nn.device_constant(params, 'bichar_embedding')
    Ec, Eb = char_table.shape[1], bichar_table.shape[1]
    # concat([char_embedding, bichar_embedding], -1): both lookups write into one buffer
    embedding = torch.empty((B, L, Ec + Eb), dtype=torch.float32, device=input_ids.device)
    ops.embedding_lookup(char_table, input_ids, out=embedding)
    ops.embedding_lookup(bichar_table, features['bichar_ids'], out=embedding, col_offset=Ec)
    return nn.bilstm_crf_tail(embedding, features, params, is_training)


TRAIN_PARAMS = dict(_BILSTM_CRF_PARAMS)
