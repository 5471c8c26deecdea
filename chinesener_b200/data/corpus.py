# -*-coding:utf-8 -*-
"""Unlabelled corpus -> masked-LM pretraining records (`python -m chinesener_b200.pretrain` reads them).

    python -m chinesener_b200.data.corpus --src a.txt[,b.txt] --out DIR --bert_dir P --max_seq_len 128 [--whole_word]
                                          [--valid_fraction 0.01] [--seed 1234]

UTF-8 text, one passage per line (blank lines skipped), is cut by `FullTokenizer` (P's vocab.txt) into consecutive chunks of
up to max_seq_len - 2 word pieces, each wrapped in [CLS] ... [SEP] (no next-sentence pairing).  DIR gets train.nerrec and
valid.nerrec with the columns token_ids, mask, segment_ids (0) and seq_len, and with --whole_word a word_start u8 column:
1 where a word of a `cut(passage) -> words` segmenter begins (jieba when installed, as SoftWordProc).  A piece starts a
word when its first character does; a character that a word piece swallowed follows its piece, and ## continuation
pieces never start a word.  There are no labels, so nothing of the NER record layout changes.
"""
import argparse
import os

import numpy as np

from . import records
from .tokenizer import BasicTokenizer, FullTokenizer


def _word_starts(text, cut):
    """Character offsets (in `text`, whitespace removed) where the segmenter's words begin."""
    words = [w for w in cut(text) if w]
    if sum(len(w) for w in words) != len(text):
        raise ValueError('segmenter output does not cover the passage {}...'.format(text[:10]))
    starts, pos = set(), 0
    for w in words:
        starts.add(pos)
        pos += len(w)
    return starts


def tokenize_passage(tokenizer, passage, cut=None):
    """-> (word pieces, word_start flags | None) of one passage."""
    basic = BasicTokenizer(do_lower_case=True)
    pieces, flags = [], []
    starts = _word_starts(''.join(passage.split()), cut) if cut is not None else None
    pos = 0                                   # character offset of the current basic token in the whitespace-free text
    for bt in basic.tokenize(passage):
        wp = tokenizer.wordpiece_tokenizer.tokenize(bt)
        used = 0
        for p in wp:
            n = len(bt) - used if p == '[UNK]' else len(p[2:] if p.startswith('##') else p)
            pieces.append(p)
            flags.append(0 if p.startswith('##') else int(starts is not None and pos + used in starts))
            used += n
        pos += len(bt)
    return pieces, (flags if cut is not None else None)


def passage_features(tokenizer, passage, max_seq_len, cut=None):
    """-> feature dicts of the passage's chunks of up to max_seq_len - 2 pieces, each [CLS] ... [SEP]."""
    pieces, flags = tokenize_passage(tokenizer, passage, cut)
    C = max_seq_len - 2
    out = []
    for s in range(0, len(pieces), C):
        toks = ['[CLS]'] + pieces[s:s + C] + ['[SEP]']
        n = len(toks)
        pad = [0] * (max_seq_len - n)
        f = {'token_ids': tokenizer.convert_tokens_to_ids(toks) + pad, 'mask': [1] * n + pad,
             'segment_ids': [0] * max_seq_len, 'seq_len': n}
        if flags is not None:
            f['word_start'] = [0] + flags[s:s + C] + [0] + pad
        out.append(f)
    return out


def build(src_files, out_dir, bert_dir, max_seq_len, cut=None, valid_fraction=0.01, seed=1234):
    """Write out_dir/train.nerrec and valid.nerrec; -> (n_train, n_valid)."""
    if max_seq_len < 3:
        raise ValueError('max_seq_len must be >= 3 ([CLS], one piece, [SEP])')
    tokenizer = FullTokenizer(os.path.join(bert_dir, 'vocab.txt'))
    feats = []
    for path in src_files:
        with open(path, encoding='utf-8') as f:
            for line in f:
                if line.strip():
                    feats += passage_features(tokenizer, line.strip(), max_seq_len, cut)
    if not feats:
        raise ValueError('no passage in {}'.format(src_files))
    order = np.random.default_rng(seed).permutation(len(feats))
    n_valid = min(len(feats) - 1, max(1, int(round(valid_fraction * len(feats))))) if valid_fraction > 0 else 0
    os.makedirs(out_dir, exist_ok=True)
    valid = [feats[i] for i in sorted(order[:n_valid])]
    train = [feats[i] for i in sorted(order[n_valid:])]
    records.write_records(os.path.join(out_dir, 'train.nerrec'), train, max_seq_len)
    records.write_records(os.path.join(out_dir, 'valid.nerrec'), valid, max_seq_len)
    return len(train), len(valid)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--src', required=True, help='comma-separated UTF-8 text files, one passage per line')
    ap.add_argument('--out', required=True)
    ap.add_argument('--bert_dir', required=True, help='directory holding vocab.txt')
    ap.add_argument('--max_seq_len', type=int, default=128)
    ap.add_argument('--whole_word', action='store_true', help='add word_start from a word segmenter (jieba)')
    ap.add_argument('--valid_fraction', type=float, default=0.01)
    ap.add_argument('--seed', type=int, default=1234)
    a = ap.parse_args(argv)
    cut = None
    if a.whole_word:
        try:
            import jieba
        except ImportError:
            raise SystemExit('--whole_word needs a word segmenter: install jieba (or call corpus.build(..., cut=...))')
        cut = jieba.cut
    n = build(a.src.split(','), a.out, a.bert_dir, a.max_seq_len, cut, a.valid_fraction, a.seed)
    print('train {} / valid {} chunks -> {}'.format(n[0], n[1], a.out))
    return n


if __name__ == '__main__':
    main()
