"""`bilstm_crf` (reference model/bilstm_crf.py:8-62): frozen pretrained character embedding -> dropout -> BiLSTM(128, tanh)
-> dropout -> label projection -> CRF."""
from .. import ops
from . import _blocks as nn

_const_table = nn.device_constant          # other plugins import the table cache under this name


def build_graph(features, labels, params, is_training):
    chars = ops.embedding_lookup(nn.device_constant(params, 'embedding'), features['token_ids'])
    return nn.bilstm_crf_tail(chars, features, params, is_training)


TRAIN_PARAMS = nn.hyper(
    dict(cell_type='lstm', cell_size=1, hidden_units_list=[128], keep_prob_list=[1], rnn_activation='tanh'),
    lr=0.005,
    decay_rate=0.95,          # lr * decay_rate ** (global_step / steps_per_epoch)
    embedding_dropout=0.3,
    early_stop_ratio=2,
)
