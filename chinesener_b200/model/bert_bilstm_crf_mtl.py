# -*-coding:utf-8 -*-
"""Plugin mirror of reference model/bert_bilstm_crf_mtl.py (build_graph :8-66, params :69-80) — SURVEY §8(f) rank 4:
one shared BertModel, one BiLSTM + logits + CRF tower per task; `task_ids` picks the tower a sentence belongs to."""
import torch

from .. import variables
from . import _blocks as nn
from ..tools.layer import bilstm, concat, crf_decode, crf_layer, dense, masked_task_loss, pretrain_bert_embedding


def _tower(embedding, label_ids, seq_len, params, task_params, is_training, extra=None):
    lstm_output = bilstm(embedding, params['cell_type'], params['rnn_activation'],
                         params['hidden_units_list'], params['keep_prob_list'],
                         params['cell_size'], seq_len, params['dtype'], is_training)
    feats = lstm_output if extra is None else concat([extra, lstm_output], is_training)
    logits = dense(feats, units=task_params['label_size'], name='logits', is_training=is_training)
    # sentences of the other task carry that task's label ids; their likelihood is masked out of the loss, the ids only
    # have to stay inside this tower's transition matrix
    labels = None if label_ids is None else label_ids.clamp(max=task_params['label_size'] - 1)
    trans, log_likelihood = crf_layer(logits, labels, seq_len, task_params['label_size'], is_training)
    pred_ids = crf_decode(logits, trans, seq_len, task_params['idx2tag'], is_training)
    return lstm_output, log_likelihood, pred_ids


def build_graph(features, labels, params, is_training):
    """
    Multi-task learning. task can be CWS + NER, or different NER dataset
    asymmetry=False, all task share bert embedding, and has its own bilstm+crf tower
    asymmetry=True, task2 is the main task, 2 task share bert embedding, task2 use task 1 hidden state also
    """
    nn.refuse_label_mask(features, 'bert_bilstm_crf_mtl')
    input_ids = features['token_ids']
    label_ids = features['label_ids']
    input_mask = features['mask']
    segment_ids = features['segment_ids']
    seq_len = features['seq_len']
    task_ids = features['task_ids']

    embedding = pretrain_bert_embedding(input_ids, input_mask, segment_ids, params['pretrain_dir'],
                                        params['embedding_dropout'], is_training)

    mask1 = task_ids == 0
    mask2 = task_ids == 1
    batch_size = task_ids.shape[0]
    with variables.variable_scope(params['task_list'][0]):
        lstm_output1, loglikelihood1, pred_ids1 = _tower(embedding, label_ids, seq_len, params,
                                                         params[params['task_list'][0]], is_training)
    with variables.variable_scope(params['task_list'][1]):
        _, loglikelihood2, pred_ids2 = _tower(embedding, label_ids, seq_len, params, params[params['task_list'][1]],
                                              is_training, extra=lstm_output1 if params['asymmetry'] else None)

    loss = masked_task_loss([loglikelihood1, loglikelihood2], [mask1, mask2], params['task_weight'], batch_size, is_training)
    pred_ids = torch.where(mask1.view(-1, 1), pred_ids1, pred_ids2)   # for inference all pred_ids will be for 1 task
    return loss, pred_ids, task_ids


TRAIN_PARAMS = nn.hyper(
    dict(cell_type='lstm', cell_size=1, hidden_units_list=[128], keep_prob_list=[0.8], rnn_activation='relu', batch_size=32),
    diff_lr_times={'crf': 500, 'logit': 500, 'lstm': 100},
    task_weight=[1, 1],       # equal weight for CWS+NER / NER+NER
    asymmetry=True,           # task 2 is the main task and also reads task 1's hidden states
)
