# -*-coding:utf-8 -*-
"""In-process counterpart of reference inference.py:33-99: `InferHelper.infer(text)` featurises one sentence exactly
like the reference's serving client and runs PREDICT on the local engine instead of a TF-Serving gRPC round trip."""
import re
from collections import defaultdict

import numpy as np

from .data.base_preprocess import extract_prefix_surfix, features_to_batch, get_instance
from .data.tokenizer import TokenizerBert
from .tools.infer_utils import extract_entity, fix_tokens

MAX_SEQ_LEN = 150
TAG2IDX = {'[PAD]': 0, 'O': 1, 'B-ORG': 2, 'I-ORG': 3, 'B-PER': 4, 'I-PER': 5, 'B-LOC': 6, 'I-LOC': 7, '[CLS]': 8, '[SEP]': 9}


class InferHelper(object):
    """`tokenizer` (and, for the word-enhance models, the keyword arguments their processor needs — the SoftLexicon word
    vocabulary) are passed in where the reference looks them up by module name; the processor class is picked from the
    model name exactly as the reference does (extract_prefix_surfix + get_instance, inference.py:36-39)."""

    def __init__(self, max_seq_len, tag2idx, model_name, tokenizer, estimator=None, **proc_kwargs):
        self.model_name = model_name
        self.word_enhance, self.tokenizer_type = extract_prefix_surfix(model_name)
        self.mtl = 1 if re.search('(mtl)|(adv)', model_name) else 0            # whether is multitask
        self.proc = get_instance(self.tokenizer_type, max_seq_len, tag2idx, tokenizer, word_enhance=self.word_enhance, **proc_kwargs)
        self.max_seq_len, self.tag2idx = max_seq_len, tag2idx
        self.idx2tag = dict((v, k) for k, v in tag2idx.items())
        self.estimator = estimator
        self.feature = None
        self.featurizer = None

    def make_feature(self, sentence):
        """reference inference.py:64-82: sequence features + fake labels ('0.0' strings / zero ids), task id for the
        multi-task models, WordPiece tokens mapped back to the sentence's characters."""
        self.feature = self.proc.build_seq_feature(sentence)
        self.feature['labels'] = np.zeros(shape=(self.max_seq_len,)).astype(str).tolist()
        self.feature['label_ids'] = np.zeros(shape=(self.max_seq_len,)).astype(int).tolist()
        if self.mtl:
            self.feature['task_ids'] = 1
        if self.tokenizer_type == TokenizerBert:
            self.feature['tokens'] = fix_tokens(sentence, self.feature['tokens'])
        return self.feature

    def decode_prediction(self, pred_ids):
        return extract_entity(self.feature['tokens'], [int(i) for i in np.squeeze(pred_ids)], self.idx2tag)

    def infer(self, text):
        feature = self.make_feature(text)
        out = self.estimator.predict(features_to_batch([feature]))
        if 'pred_spans' in out:                  # span-pointer plugin: every (possibly nested) span, not the tag scan
            from .tools.infer_utils import span_entities
            return span_entities([feature['tokens']], out['pred_spans'])[0]
        return self.decode_prediction(out['pred_ids'].numpy())

    def infer_nbest(self, text):
        """The estimator's params['crf_nbest'] best CRF paths of one sentence -> a list of (entity dict, probability), best
        first, one entry per path; the first entity dict is infer(text).  Entries are not merged: two paths that give the
        same entities (for example paths that differ only at [CLS] / [SEP]) are two entries, each with its own
        probability exp(score - log Z)."""
        import torch
        from .tools.infer_utils import extract_entity_device
        feature = self.make_feature(text)
        out = self.estimator.predict(features_to_batch([feature]))
        if 'pred_nbest' not in out:
            raise ValueError(f"infer_nbest needs a CRF plugin run with params['crf_nbest'] > 1 ({self.model_name})")
        paths = out['pred_nbest'][0]
        if not paths:
            return []
        rows = torch.from_numpy(np.stack([p[0] for p in paths])).to(self.estimator.device)
        ents = extract_entity_device([feature['tokens']] * len(paths), rows, self.idx2tag)
        return [(e, p[2]) for e, p in zip(ents, paths)]

    def infer_batch(self, texts):
        """Many sentences per call: one PREDICT batch, the tag scan of extract_entity on the GPU (ner_extract_spans) —
        the tag tensor stays on the device, only the spans come back.  -> one entity dict per text, as infer() gives.
        A span-pointer plugin (bert_mrc_span) returns its own spans instead, nested and overlapping ones included.

        Plugins whose features are BasicProc's alone (no word-enhance method) featurise the raw texts on the device
        (data/device_featurize.py, built on first use and kept), and the entity strings are rebuilt for the returned
        spans only; the word-enhance plugins featurise on the host with make_feature."""
        import torch
        from .tools.infer_utils import extract_entity_device, span_entities, span_lists, tag_spans_device
        if self.word_enhance is not None or not texts:
            feats = [dict(self.make_feature(t)) for t in texts]
            dev = self.estimator.to_device(features_to_batch(feats, pin_memory=True))
            pred = self.estimator.predict_device(dev)
            spans = span_lists(pred)
            if spans is not None:
                return span_entities([f['tokens'] for f in feats], spans)
            return extract_entity_device([f['tokens'] for f in feats], pred, self.idx2tag)
        if self.featurizer is None:
            from .data.device_featurize import DeviceFeaturizer
            self.featurizer = DeviceFeaturizer(self.proc.tokenizer, self.max_seq_len, self.estimator.device)
        dev = self.featurizer.featurize(texts, task_id=1 if self.mtl else None)
        host = {}
        for k in ('token_ids', 'unk_cursor'):        # read only for the spans' strings, after the span scan's sync
            host[k] = torch.empty(dev[k].shape, dtype=torch.int32, pin_memory=True)
            host[k].copy_(dev[k], non_blocking=True)
        del dev['unk_cursor']
        pred = self.estimator.predict_device(dev)
        spans = span_lists(pred)
        if spans is None:
            spans = tag_spans_device(pred, self.idx2tag)
        text = self.featurizer.entity_text(texts, host['token_ids'].numpy(), host['unk_cursor'].numpy(),
                                           dev['mask'].row_lengths)
        out = []
        for b, row in enumerate(spans):
            found = defaultdict(set)
            for span in row:
                s = text(b, span[1], span[2])
                if s != '':
                    found[span[0]].add(s)
            out.append(found)
        return out
