# -*-coding:utf-8 -*-
"""Entity / tag level evaluation of `<model>_predict.pkl` files (reference evaluation.py).

seqeval and sklearn reports are restated here (seqeval is not installable offline):
`get_entities` follows seqeval's default (non-strict) chunking rules, the report is
per-type precision / recall / F1 with micro and support-weighted averages — the numbers
evaluation.py:48-55,86-93 prints.
"""
import pickle
from collections import defaultdict

import numpy as np

from .tools.predict_utils import process_prediction


def _end_of_chunk(prev_tag, tag, prev_type, type_):
    if prev_tag in ('E', 'S'):
        return True
    if prev_tag in ('B', 'I') and tag in ('B', 'S', 'O'):
        return True
    return prev_tag not in ('O', '.') and prev_type != type_


def _start_of_chunk(prev_tag, tag, prev_type, type_):
    if tag in ('B', 'S'):
        return True
    if prev_tag in ('E', 'S', 'O') and tag in ('E', 'I'):
        return True
    return tag not in ('O', '.') and prev_type != type_


def get_entities(seq):
    """seqeval.metrics.sequence_labeling.get_entities over a list of tag lists."""
    if any(isinstance(s, list) for s in seq):
        seq = [item for sub in seq for item in sub + ['O']]
    prev_tag, prev_type, begin = 'O', '', 0
    chunks = []
    for i, chunk in enumerate(seq + ['O']):
        tag = chunk[0]
        type_ = chunk.split('-', 1)[-1] if '-' in chunk else ('' if tag == 'O' else chunk)
        if _end_of_chunk(prev_tag, tag, prev_type, type_):
            chunks.append((prev_type, begin, i - 1))
        if _start_of_chunk(prev_tag, tag, prev_type, type_):
            begin = i
        prev_tag, prev_type = tag, type_
    return chunks


def entity_report(y_true, y_pred):
    """-> {type: {precision, recall, f1-score, support}, 'micro avg': ..., 'weighted avg': ...}."""
    true_e, pred_e = set(get_entities(y_true)), set(get_entities(y_pred))
    by_t, by_p = defaultdict(set), defaultdict(set)
    for e in true_e:
        by_t[e[0]].add(e)
    for e in pred_e:
        by_p[e[0]].add(e)
    rep = {}

    def prf(tp, npred, ntrue):
        p = tp / npred if npred else 0.0
        r = tp / ntrue if ntrue else 0.0
        f = 2 * p * r / (p + r) if p + r else 0.0
        return {'precision': p, 'recall': r, 'f1-score': f, 'support': ntrue}

    for t in sorted(set(by_t) | set(by_p)):
        rep[t] = prf(len(by_t[t] & by_p[t]), len(by_p[t]), len(by_t[t]))
    rep['micro avg'] = prf(len(true_e & pred_e), len(pred_e), len(true_e))
    tot = sum(v['support'] for k, v in rep.items() if k != 'micro avg')
    rep['weighted avg'] = {m: (sum(v[m] * v['support'] for k, v in rep.items() if k != 'micro avg') / tot if tot else 0.0)
                           for m in ('precision', 'recall', 'f1-score')}
    rep['weighted avg']['support'] = tot
    return rep


def tag_report(y_true, y_pred, labels):
    """sklearn-style per-tag precision/recall/F1 + weighted average over `labels` (tag ids)."""
    rep = {}
    for lab in labels:
        tp = sum(1 for a, b in zip(y_true, y_pred) if a == lab and b == lab)
        npred = sum(1 for b in y_pred if b == lab)
        ntrue = sum(1 for a in y_true if a == lab)
        p = tp / npred if npred else 0.0
        r = tp / ntrue if ntrue else 0.0
        rep[lab] = {'precision': p, 'recall': r, 'f1-score': 2 * p * r / (p + r) if p + r else 0.0, 'support': ntrue}
    tot = sum(v['support'] for v in rep.values())
    rep['weighted avg'] = {m: sum(v[m] * v['support'] for v in rep.values()) / tot if tot else 0.0
                           for m in ('precision', 'recall', 'f1-score')}
    return rep


class SingleEval(object):
    """reference evaluation.py:16-75 over an in-memory prediction list or a pickle path."""

    def __init__(self, prediction, idx2tag, verbose=False):
        if isinstance(prediction, str):
            with open(prediction, 'rb') as f:
                prediction = pickle.load(f)
        self.idx2tag = idx2tag
        for i in prediction:
            if (np.asarray(i['label_ids']) < 0).any():
                raise ValueError('SingleEval needs gold tags at every position; this prediction carries partial labels '
                                 '(label_id -1 at open positions), whose gold entities are unknown')
        self.prediction = [process_prediction(dict(i), idx2tag) for i in prediction]
        self.verbose = verbose

    def entity_eval(self):
        return entity_report([i['labels'] for i in self.prediction], [i['preds'] for i in self.prediction])

    def tag_eval(self):
        y_true = [int(t) for i in self.prediction for t in i['label_ids']]
        y_pred = [int(t) for i in self.prediction for t in i['pred_ids']]
        labels = [k for k, v in self.idx2tag.items() if v not in ('[PAD]', '[CLS]', '[SEP]')]
        return tag_report(y_true, y_pred, labels)

    def gen_report(self):
        return self.tag_eval(), self.entity_eval()
