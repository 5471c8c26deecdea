# -*-coding:utf-8 -*-
"""Feature-dict builder with the reference's surface (reference data/base_preprocess.py:137-227, BasicProc) minus the
TFRecord writer: one sentence -> {'tokens','token_ids','segment_ids','mask','seq_len'[, 'labels','label_ids']} padded to
max_seq_len, and `features_to_batch` -> the int32 tensor dict the plugins' build_graph consumes (dataset.py:21-37)."""
import re

import torch

from .tokenizer import TokenizerBert, TokenizerGiga

SoftWord, ExSoftWord, SoftLexicon, BiChar, Lattice = 'softword', 'ex_softword', 'softlexicon', 'bichar', 'lattice'
WordEnhanceMethod = [SoftWord, ExSoftWord, SoftLexicon, BiChar, Lattice]


def extract_prefix_surfix(model_name):
    """-> (word_enhance, tokenizer_type) from the model name (reference :25-36): a name containing 'bert' uses the BERT
    tokenizer, else giga; the word-enhance method is the first of softword / softlexicon / ex_softword / bichar / lattice
    the alternation finds (leftmost match, alternatives tried in that order — 'ex_softword' names match 'softword' only
    when no earlier position matches, exactly as the reference's regex does; 'lattice' comes last, so every name without
    it maps as the reference maps it)."""
    m = re.search('({})|({})|({})|({})|({})'.format(SoftWord, SoftLexicon, ExSoftWord, BiChar, Lattice), model_name)
    word_enhance = m.group() if m else None
    tokenizer_type = TokenizerBert if re.search('({})'.format(TokenizerBert), model_name) else TokenizerGiga
    return word_enhance, tokenizer_type


def get_instance(tokenizer_type, max_seq_len, tag2idx, tokenizer, word_enhance=None, **kwargs):
    """reference :75-93 — the processor class for a word-enhance method (None -> BasicProc, softlexicon ->
    SoftLexiconProc(vocab), bichar -> BiCharProc(bichar_tokenizer), softword -> SoftWordProc(cut), ex_softword ->
    ExSoftWordProc(vocab), lattice -> LatticeProc(vocab, word_embedding)); the tokenizer object and the method's keyword
    arguments are passed in instead of being looked up by name because vocabularies / vectors live wherever the caller
    keeps them."""
    assert word_enhance in [None] + WordEnhanceMethod, 'word_enhance must in {}'.format(','.join(WordEnhanceMethod))
    if word_enhance is None:
        return BasicProc(tokenizer_type, max_seq_len, tag2idx, tokenizer)
    from . import word_enhance as we
    cls = {SoftLexicon: we.SoftLexiconProc, BiChar: we.BiCharProc, SoftWord: we.SoftWordProc,
           ExSoftWord: we.ExSoftWordProc, Lattice: we.LatticeProc}[word_enhance]
    return cls(tokenizer_type, max_seq_len, tag2idx, tokenizer, **kwargs)


SPECIAL_TAGS = ('[PAD]', '[CLS]', '[SEP]')
OPEN_TAG, TAG_SET_SEP = '?', '|'


def tag_set_mask(tag, tag2idx):
    """The allowed-tag bitmask of one partial label: '?' allows every tag a real token may carry (all but [PAD], [CLS]
    and [SEP]), 'T1|T2|...' the listed tags.  A set naming an unknown or special tag raises ValueError.  Returned as a
    signed int32 value (bit 31, tag id 31, is the sign bit)."""
    if tag == OPEN_TAG:
        ids = [i for t, i in tag2idx.items() if t not in SPECIAL_TAGS]
    else:
        names = tag.split(TAG_SET_SEP)
        bad = [t for t in names if t not in tag2idx or t in SPECIAL_TAGS]
        if bad:
            raise ValueError('tag set {!r}: unknown or special tag {}'.format(tag, ', '.join(map(repr, bad))))
        ids = [tag2idx[t] for t in names]
    return _bits(ids)


def _bits(ids):
    """tag ids -> the int32 bitmask with those bits set (bit 31 as the sign bit)."""
    if any(not 0 <= i < 32 for i in ids):
        raise ValueError('a label_mask holds tag ids below 32 only, got {}'.format(sorted(ids)))
    m = sum(1 << i for i in set(ids))
    return m - (1 << 32) if m >= 1 << 31 else m


class BasicProc(object):
    # partial_labels: tags.txt may hold '?' / 'T1|T2|...' entries (build_tag_feature); set by the preprocess CLI
    partial_labels = False

    def __init__(self, tokenizer_type, max_seq_len, tag2idx, tokenizer):
        assert tokenizer_type in (TokenizerBert, TokenizerGiga)
        self.tokenizer_type, self.max_seq_len, self.tag2idx, self.tokenizer = tokenizer_type, max_seq_len, tag2idx, tokenizer

    def format_sequence(self, seq):
        """Bert: [CLS] + seq[:L-2] + [SEP], then [PAD]; non-bert: seq[:L], then [PAD]   (reference :164-177)."""
        seq = list(seq)
        if self.tokenizer_type == TokenizerBert:
            seq = ['[CLS]'] + seq[:(self.max_seq_len - 2)] + ['[SEP]']
        else:
            seq = seq[:self.max_seq_len]
        seq_len = len(seq)
        seq += ['[PAD]'] * (self.max_seq_len - seq_len)
        return seq, seq_len

    def build_seq_feature(self, sentence):
        tokens = self.tokenizer.tokenize(sentence)
        tokens, seq_len = self.format_sequence(tokens)
        token_ids = self.tokenizer.convert_tokens_to_ids(tokens)
        segment_ids = [0] * self.max_seq_len
        mask = [1] * seq_len + [0] * (self.max_seq_len - seq_len)
        assert len(tokens) == len(token_ids) == len(mask) == self.max_seq_len
        return {'tokens': tokens, 'token_ids': token_ids, 'segment_ids': segment_ids, 'mask': mask, 'seq_len': seq_len}

    def build_tag_feature(self, tag):
        """With partial_labels, an entry of `tag` may be a tag set ('?' or 'T1|T2|...'): it gets label_id -1, and the
        `label_mask` row holds every position's allowed-tag bitmask (the one-hot bit of its label_id elsewhere, [CLS],
        [SEP] and [PAD] included)."""
        labels, label_len = self.format_sequence(tag.split(' '))
        if not self.partial_labels:
            label_ids = [self.tag2idx[i] for i in labels]
            return {'labels': labels, 'label_ids': label_ids, 'label_len': label_len}
        label_ids, label_mask = [], []
        for t in labels:
            if t == OPEN_TAG or TAG_SET_SEP in t:
                label_ids.append(-1)
                label_mask.append(tag_set_mask(t, self.tag2idx))
            else:
                label_ids.append(self.tag2idx[t])
                label_mask.append(_bits([label_ids[-1]]))
        return {'labels': labels, 'label_ids': label_ids, 'label_mask': label_mask, 'label_len': label_len}

    def build_feature(self, sentence, tag):
        f_seq, f_label = self.build_seq_feature(sentence), self.build_tag_feature(tag)
        assert f_seq['seq_len'] == f_label['label_len'], \
            'sentence = {}... {}!={} n_token!=n_tag'.format(sentence[:10], f_seq['seq_len'], f_label['label_len'])
        return {**f_seq, **f_label}

    def build_data_params(self, n_sample):
        """reference :206-222 (the giga `embedding` entry is added by the caller that owns the vectors)."""
        return {'n_sample': n_sample, 'max_seq_len': self.max_seq_len, 'label_size': len(self.tag2idx), 'tag2idx': self.tag2idx,
                'idx2tag': dict((v, k) for k, v in self.tag2idx.items())}


def features_to_batch(features, pin_memory=False):
    """list of feature dicts -> the batched int32 tensors of dataset.py:21-37 (strings stay host-side lists)."""
    L = len(features[0]['token_ids'])
    out = {k: torch.tensor([f[k] for f in features], dtype=torch.int32) for k in ('token_ids', 'mask', 'segment_ids')}
    out['seq_len'] = torch.tensor([f['seq_len'] for f in features], dtype=torch.int32)
    out['label_ids'] = torch.tensor([f.get('label_ids', [0] * L) for f in features], dtype=torch.int32)
    if 'label_mask' in features[0]:     # partially annotated sentences (BasicProc.build_tag_feature)
        out['label_mask'] = torch.tensor([f['label_mask'] for f in features], dtype=torch.int32)
    # optional per-plugin features (dataset.py:29-36, MultiDataset.add_discriminator :88-90)
    for k in ('softlexicon_ids', 'bichar_ids', 'softword_ids', 'lattice_ids', 'lattice_lens'):
        if k in features[0]:
            out[k] = torch.tensor([f[k] for f in features], dtype=torch.int32)
    for k in ('softlexicon_weights', 'ex_softword_ids'):
        if k in features[0]:
            out[k] = torch.tensor([f[k] for f in features], dtype=torch.float32)
    if 'task_ids' in features[0]:      # one task id per sentence (serving receiver: FixedLenFeature([], int64), infer_utils.py:60-63)
        out['task_ids'] = torch.tensor([int(f['task_ids']) for f in features], dtype=torch.int32)
    if pin_memory:
        out = {k: v.pin_memory() for k, v in out.items()}
    out['tokens'] = [f['tokens'] for f in features]
    out['labels'] = [f.get('labels') for f in features]
    return out
