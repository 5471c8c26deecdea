# -*-coding:utf-8 -*-
"""Plugin mirror of reference model/bert_bilstm_crf_adv.py (build_graph :9-87, params :90-107) — SURVEY §8(f) rank 4:
shared BertModel -> a shared BiLSTM read by a task discriminator through max-pool + gradient flip, and one private
BiLSTM + logits + CRF tower per task over [shared | private] hidden states.

The reference's task-2 tower calls bilstm() without seq_len (:68-70, one positional argument short), so the upstream
file cannot build its graph as written; this mirror passes seq_len there as the task-1 tower (:51-53) does."""
import torch

from .. import variables
from . import _blocks as nn
from ..tools.layer import (bilstm, concat, crf_decode, crf_layer, dense, dropout, masked_task_loss,
                           pretrain_bert_embedding, reduce_max_flip, softmax_cross_entropy_mean)


def build_graph(features, labels, params, is_training):
    """
    Adversarial Training. task can be CWS + NER, or different NER dataset
    all task share bert embedding, and has its own bilstm+crf layer
    Equal weight for all task, with lambda weight for discriminator
    """
    nn.refuse_label_mask(features, 'bert_bilstm_crf_adv')
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

    def _bilstm():
        return bilstm(embedding, params['cell_type'], params['rnn_activation'],
                      params['hidden_units_list'], params['keep_prob_list'],
                      params['cell_size'], seq_len, params['dtype'], is_training)

    with variables.variable_scope('task_discriminator'):
        share_output = _bilstm()  # batch * max_seq * (2*hidden)
        # extract most significant feature; the reversed (and shrunk) gradient only updates the units used to tell tasks apart
        share_max_pool = reduce_max_flip(share_output, params['shrink_gradient_reverse'], is_training)
        share_max_pool = dropout(share_max_pool, params['share_dropout'], is_training, seed=1234)
        logits = dense(share_max_pool, units=len(params['task_list']), name='logits', is_training=is_training)  # batch * num_task
        adv_loss = softmax_cross_entropy_mean(logits, task_ids, params['lambda'], is_training)

    log_likelihoods, preds = [], []
    for t, task in enumerate(params['task_list'][:2]):
        with variables.variable_scope('task{}_{}'.format(t + 1, task)):
            task_params = params[task]
            lstm_output = concat([share_output, _bilstm()], is_training)  # batch * (4*hidden)
            logits = dense(lstm_output, units=task_params['label_size'], name='logits', is_training=is_training)
            tower_labels = None if label_ids is None else label_ids.clamp(max=task_params['label_size'] - 1)
            trans, ll = crf_layer(logits, tower_labels, seq_len, task_params['label_size'], is_training)
            preds.append(crf_decode(logits, trans, seq_len, task_params['idx2tag'], is_training))
            log_likelihoods.append(ll)

    loss = masked_task_loss(log_likelihoods, [mask1, mask2], params['task_weight'], batch_size, is_training) + adv_loss
    pred_ids = torch.where(mask1.view(-1, 1), preds[0], preds[1])
    return loss, pred_ids, task_ids


TRAIN_PARAMS = nn.hyper(
    dict(cell_type='lstm', cell_size=1, hidden_units_list=[100], keep_prob_list=[0.8], rnn_activation='relu'),
    diff_lr_times={'crf': 500, 'logit': 100, 'lstm': 100},
    task_weight=[1, 1],
    share_dropout=0.2,
    shrink_gradient_reverse=0.001,     # the reference suggests 0.01 for CWS+NER, 0.001 for NER+NER
    batch_size=32,
    **{'lambda': 0.5},                 # weight of the task-discriminator loss
)
