"""`bert_ce` (reference model/bert_ce.py): BertModel sequence output -> label projection -> softmax, trained with the
masked token cross-entropy of tools/loss.py; pred_ids = tf.argmax(logits, -1) at every position.

PREDICT / EVAL run the encoder on the padded layout: the reference's argmax is not masked, so a [PAD] position gets the
tag of BertModel's real output there (a [PAD] row is a query over the valid keys), and its prediction pickles carry
those non-zero tags.  TRAIN uses the packed encoder: the loss reads only t < seq_len, so packing is exact for the loss
and every gradient.

params['bert_precision'] = 'fp32' runs the fp32-accurate encoder, whose attention writes zero rows for [PAD] queries: the
loss and the tags of the real tokens are unaffected, the [PAD] tags are then not the reference's."""
from ..tools import layer as L
from ..tools.loss import argmax, cross_entropy_loss
from . import _blocks as nn


def build_graph(features, labels, params, is_training):
    nn.refuse_label_mask(features, 'bert_ce')
    hidden = nn.bert_sequence(features, params, is_training, packed=is_training)
    logits = L.dense(hidden, units=params['label_size'], name='logits', is_training=is_training)
    loss = cross_entropy_loss(logits, features.get('label_ids'), features['seq_len'], params['max_seq_len'], is_training)
    pred_ids = loss.pred_ids if is_training else argmax(logits)
    return loss, pred_ids


# bert_crf's recipe without the 'crf' group (the reference's bert_ce parameters are not in this repository: unpinned)
TRAIN_PARAMS = nn.hyper(diff_lr_times={'logit': 500})
