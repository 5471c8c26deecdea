"""`bert_dice` (reference model/bert_dice.py): bert_ce's graph — BertModel sequence output -> label projection ->
softmax, pred_ids = tf.argmax(logits, -1) at every position — trained with the self-adjusting Dice loss of tools/loss.py
instead of the cross-entropy.

PREDICT / EVAL run the encoder on the padded layout and TRAIN on the packed one, for the reasons model/bert_ce.py gives:
the argmax covers the [PAD] positions, the loss reads only t < seq_len.  params['dice_alpha'] (the (1-p)^alpha weight)
and params['dice_gamma'] (the smoothing term) parameterise the loss."""
from ..tools import layer as L
from ..tools.loss import argmax, dice_loss
from . import _blocks as nn


def build_graph(features, labels, params, is_training):
    nn.refuse_label_mask(features, 'bert_dice')
    hidden = nn.bert_sequence(features, params, is_training, packed=is_training)
    logits = L.dense(hidden, units=params['label_size'], name='logits', is_training=is_training)
    loss = dice_loss(logits, features.get('label_ids'), features['seq_len'], params['max_seq_len'], params['dice_alpha'],
                     params['dice_gamma'], is_training)
    pred_ids = loss.pred_ids if is_training else argmax(logits)
    return loss, pred_ids


# bert_ce's recipe; the reference's bert_dice parameters and its tools/loss.py are not in this repository, so the loss
# defaults (alpha = 1: the paper's (1-p)·p weighting, gamma = 1) are unpinned, as the 'logit' learning-rate factor is
TRAIN_PARAMS = nn.hyper(diff_lr_times={'logit': 500}, dice_alpha=1.0, dice_gamma=1.0)
