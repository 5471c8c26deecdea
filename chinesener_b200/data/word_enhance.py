# -*-coding:utf-8 -*-
"""Word-enhance featurisation of the giga character models: SoftLexicon, and the BiChar / Softword / ExSoftword inputs.

BiChar / Softword / ExSoftword (`BiCharProc`, `SoftWordProc`, `ExSoftWordProc`, after Ma et al., "Simplify the Usage of
Lexicon in Chinese NER", ACL 2020, and the bigram input of TENER) are restatements: the reference's own
data/word_enhance.py is not in this repository, so the bigram end marker, the segmentation label-to-id maps and the
ExSoftword multi-hot layout below are this project's choices, not pinned to it.  All three follow the giga tokenizer's
characters (whitespace dropped); word-piece alignment for the BERT tokenizer is not built.

SoftLexicon host side (SURVEY §8(f) rank 3) — the step just before the gather-and-pool kernel (ner_softlexicon_pool_fwd).

The matching itself (reference data/word_enhance.py:302-337 build_soft_lexicon, :89-119 align_with_token, :163-205
postproc_soft_lexicon, data/base_preprocess.py:397-412 format_soft_seq) runs in C++ behind the C-ABI
(`ner_lexicon_create / ner_lexicon_build`, chinesener_b200/csrc/lexicon_host.cu): a code-point trie over the word
vocabulary, whole lists of sentences per call on a pool of host threads, output already in the kernel's
[n, max_seq_len * 40] id / weight layout.  This module keeps the reference's Python surface around it: `WordVocab` (the word
side of VocabModel, :36-70) and `SoftLexiconProc` (data/base_preprocess.py:376-438).  The Python restatement of the reference
loop lives in oracle/lexicon.py and is only the tests' checker.
"""
import numpy as np

from .base_preprocess import BasicProc
from .tokenizer import TokenizerBert

MaxWordLen = 10
MaxLexiconLen = 10      # only keep top-n words per B/M/E/S set
SoftKeys = ('B', 'M', 'E', 'S')
MaxLatticeWords = 4     # lattice words kept per start character (the most frequent)


class WordVocab(object):
    """The word side of reference VocabModel (:36-70): vocabulary order = embedding row, add-on tokens <None> = n_word,
    <PAD> = n_word + 1, <eos> = n_word + 2; frequencies from the pretrained model, <None> -> 1, <PAD> -> 0."""
    none_token, pad_token, eos_token = '<None>', '<PAD>', '<eos>'

    def __init__(self, index2word, counts):
        self.index2word = list(index2word)
        self.vocab2idx = dict((w, i) for i, w in enumerate(self.index2word))
        self.vocab_freq = dict((self.vocab2idx[w], counts[w]) for w in self.index2word)
        self.n_word = len(self.vocab_freq)
        self.vocab2idx.update({self.none_token: self.n_word, self.pad_token: self.n_word + 1, self.eos_token: self.n_word + 2})
        self.vocab_freq.update({self.vocab2idx[self.none_token]: 1, self.vocab2idx[self.pad_token]: 0})


def _utf32(strings):
    """list of str -> (uint32 code points back to back, int64 offsets [n + 1])."""
    offs = np.zeros(len(strings) + 1, np.int64)
    np.cumsum([len(s) for s in strings], out=offs[1:])
    cps = np.frombuffer(''.join(strings).encode('utf-32-le'), dtype=np.uint32)
    assert cps.size == offs[-1]
    return np.ascontiguousarray(cps), offs


def token_char_lens(tokens):
    """characters each WordPiece token covers (reference align_with_token :94): '##' stripped, [UNK] = 1, specials skipped."""
    return [len(t.replace('##', '')) if t != '[UNK]' else 1 for t in tokens if t not in ('[CLS]', '[SEP]', '[PAD]')]


class NativeLexicon(object):
    """The vocabulary as a C++ trie.  `vocabfreq` (id -> frequency, default the vocabulary's own counts) is what
    postproc_soft_lexicon weighs by; ids it does not hold weigh 1 (`vocabfreq.get(i, 1)`, reference :182)."""

    def __init__(self, vocab, vocabfreq=None):
        from .. import _lib
        self._lib = _lib.lib()
        self.vocab, self.n_word = vocab, vocab.n_word
        words = getattr(vocab, 'index2word', None)
        if words is None:
            words = [w for w, i in sorted(vocab.vocab2idx.items(), key=lambda kv: kv[1]) if i < vocab.n_word]
        freq_of = vocab.vocab_freq if vocabfreq is None else vocabfreq
        freq = np.asarray([freq_of.get(i, 1) for i in range(self.n_word + 2)], dtype=np.float64)
        cps, offs = _utf32(words)
        self._h = self._lib.ner_lexicon_create(cps.ctypes.data, offs.ctypes.data, freq.ctypes.data, self.n_word)
        if not self._h:
            raise _lib.NerB200Error('ner_lexicon_create failed (bad vocabulary input)')

    def __del__(self):
        h, self._h = getattr(self, '_h', None), None
        if h:
            self._lib.ner_lexicon_destroy(h)

    def num_nodes(self):
        return int(self._lib.ner_lexicon_num_nodes(self._h))

    def build(self, sentences, max_seq_len, bert=False, tokens=None, n_threads=0):
        """sentences: list of raw strings; tokens (bert only): per sentence the tokenizer's tokens, so that rows follow the
        word pieces.  -> (ids int32 [n, max_seq_len * 40], weights float32 [n, max_seq_len * 40])."""
        from .. import _lib
        n = len(sentences)
        cps, offs = _utf32([s.replace(' ', '') for s in sentences])
        tl = toff = None
        if bert and tokens is not None:
            lens = [token_char_lens(t) for t in tokens]
            toff = np.zeros(n + 1, np.int64)
            np.cumsum([len(x) for x in lens], out=toff[1:])
            tl = np.asarray([v for x in lens for v in x], dtype=np.int32)
        ids = np.empty((n, max_seq_len * len(SoftKeys) * MaxLexiconLen), np.int32)
        wts = np.empty(ids.shape, np.float32)
        if tl is not None and tl.size == 0:
            tl = np.zeros(1, np.int32)          # keep the pointer non-NULL: "token lengths given, all sentences empty"
        _lib.check(self._lib.ner_lexicon_build(
            self._h, cps.ctypes.data if cps.size else None, offs.ctypes.data, n, None if tl is None else tl.ctypes.data,
            None if toff is None else toff.ctypes.data, max_seq_len, 1 if bert else 0, ids.ctypes.data, wts.ctypes.data, n_threads))
        _lib.LAUNCHES -= 1          # host call, not a kernel launch
        return ids, wts

    def build_lattice(self, sentences, max_seq_len, max_words=MaxLatticeWords, n_threads=0):
        """Lattice word lists (ner_lexicon_build_lattice): sentences are lists of characters (or strings, one character per
        position).  -> (ids int32 [n, max_seq_len * max_words], lens int32 [n, max_seq_len * max_words], number of matches
        the max_words cap dropped)."""
        from .. import _lib
        n = len(sentences)
        cps, offs = _utf32([''.join(s) for s in sentences])
        ids = np.empty((n, max_seq_len * max_words), np.int32)
        lens = np.empty(ids.shape, np.int32)
        dropped = np.zeros(1, np.int64)
        _lib.check(self._lib.ner_lexicon_build_lattice(
            self._h, cps.ctypes.data if cps.size else None, offs.ctypes.data, n, max_seq_len, max_words, ids.ctypes.data,
            lens.ctypes.data, dropped.ctypes.data, n_threads))
        _lib.LAUNCHES -= 1          # host call, not a kernel launch
        return ids, lens, int(dropped[0])


class SoftLexiconProc(BasicProc):
    """BasicProc + softlexicon_ids / softlexicon_weights (one lexicon row per token; word pieces merge their characters).
    `build_seq_features(sentences)` featurises a list in one native call; `build_seq_feature` is the reference's
    one-sentence surface over it."""

    def __init__(self, tokenizer_type, max_seq_len, tag2idx, tokenizer, vocab, vocabfreq=None):
        super(SoftLexiconProc, self).__init__(tokenizer_type, max_seq_len, tag2idx, tokenizer)
        self.vocab, self.vocabfreq = vocab, vocabfreq
        self.word_enhance = 'softlexicon'
        self.lexicon = NativeLexicon(vocab, vocabfreq)

    def build_seq_features(self, sentences, n_threads=0):
        feats = [super(SoftLexiconProc, self).build_seq_feature(s) for s in sentences]
        bert = self.tokenizer_type == TokenizerBert
        ids, wts = self.lexicon.build(sentences, self.max_seq_len, bert, [f['tokens'] for f in feats] if bert else None, n_threads)
        for f, i, w in zip(feats, ids, wts):
            f['softlexicon_ids'], f['softlexicon_weights'] = i.tolist(), w.tolist()
        return feats

    def build_seq_feature(self, sentence):
        return self.build_seq_features([sentence], n_threads=1)[0]

    def build_data_params(self, n_sample):
        params = super(SoftLexiconProc, self).build_data_params(n_sample)
        params.update({'word_enhance_dim': len(SoftKeys), 'max_lexicon_len': MaxLexiconLen, 'vocab2idx': self.vocab.vocab2idx})
        return params


# ----------------------------------------------------------------------------- BiChar / Softword / ExSoftword
BiCharEnd = '-null-'                 # pairs with the last character (the end key of the giga bigram vectors' convention)
SoftWordIds = {'B': 1, 'M': 2, 'E': 3, 'S': 4}        # softword_ids; 0 = no label / [PAD]
ExSoftWordKeys = SoftKeys + ('None',)                   # ex_softword_ids columns


def giga_chars(sentence):
    """The characters the giga tokenizer keeps (whitespace dropped), full-width folded as TokenizerAdapter does."""
    from .tokenizer import TokenizerAdapter
    return [TokenizerAdapter.full2half(c) for c in sentence if c.strip()]


def _reject_bert(tokenizer_type, name):
    if tokenizer_type == TokenizerBert:
        raise ValueError('{} follows the giga tokenizer\'s characters; BERT word-piece alignment is not built'.format(name))


class BiCharProc(BasicProc):
    """BasicProc + bichar_ids [L] int32: character j's bigram is c_j c_{j+1}, the last character's is c_n + '-null-'.
    `bichar_tokenizer` is a TokenizerAdapter over bigram vectors (get_giga_tokenizer(<bigram .vec>)): out-of-vocabulary
    bigrams are [UNK], positions past seq_len [PAD].  The caller stores the bigram table as params['bichar_embedding']."""

    def __init__(self, tokenizer_type, max_seq_len, tag2idx, tokenizer, bichar_tokenizer):
        _reject_bert(tokenizer_type, 'BiCharProc')
        super(BiCharProc, self).__init__(tokenizer_type, max_seq_len, tag2idx, tokenizer)
        self.bichar_tokenizer = bichar_tokenizer
        self.word_enhance = 'bichar'

    def bigrams(self, sentence):
        chars = giga_chars(sentence)
        vocab = self.bichar_tokenizer.vocab2idx
        grams = [a + b for a, b in zip(chars, chars[1:] + [BiCharEnd])]
        return [g if g in vocab else '[UNK]' for g in grams]

    def build_seq_feature(self, sentence):
        f = super(BiCharProc, self).build_seq_feature(sentence)
        grams, _ = self.format_sequence(self.bigrams(sentence))
        f['bichar_ids'] = self.bichar_tokenizer.convert_tokens_to_ids(grams)
        return f


def ex_softword_from_lexicon(ids, seq_len, none_id, max_seq_len):
    """NativeLexicon.build ids [n, L * 40] -> ex_softword_ids float32 [n, L * 5]: per character the multi-hot of the
    B/M/E/S sets its lexicon match holds (a set is non-empty when its first slot is not <None>), None when all four are
    empty; rows at or past seq_len are zero."""
    n = ids.shape[0]
    first = ids.reshape(n, max_seq_len, len(SoftKeys), MaxLexiconLen)[..., 0]          # [n, L, 4]
    out = np.zeros((n, max_seq_len, len(ExSoftWordKeys)), np.float32)
    out[..., :len(SoftKeys)] = first != none_id
    out[..., len(SoftKeys)] = ~out[..., :len(SoftKeys)].any(-1)
    out[np.arange(max_seq_len)[None, :] >= np.asarray(seq_len)[:, None]] = 0
    return out.reshape(n, -1)


class ExSoftWordProc(BasicProc):
    """BasicProc + ex_softword_ids [L * 5] float32 (ExSoftword: the multi-hot B/M/E/S/None label set of every character,
    from the SoftLexicon match against `vocab`, a WordVocab)."""

    def __init__(self, tokenizer_type, max_seq_len, tag2idx, tokenizer, vocab, vocabfreq=None):
        _reject_bert(tokenizer_type, 'ExSoftWordProc')
        super(ExSoftWordProc, self).__init__(tokenizer_type, max_seq_len, tag2idx, tokenizer)
        self.vocab, self.word_enhance = vocab, 'ex_softword'
        self.lexicon = NativeLexicon(vocab, vocabfreq)

    def build_seq_features(self, sentences, n_threads=0):
        feats = [super(ExSoftWordProc, self).build_seq_feature(s) for s in sentences]
        ids, _ = self.lexicon.build(sentences, self.max_seq_len, False, None, n_threads)
        ex = ex_softword_from_lexicon(ids, [f['seq_len'] for f in feats], self.vocab.vocab2idx[WordVocab.none_token],
                                      self.max_seq_len)
        for f, x in zip(feats, ex):
            f['ex_softword_ids'] = x.tolist()
        return feats

    def build_seq_feature(self, sentence):
        return self.build_seq_features([sentence], n_threads=1)[0]


class LatticeProc(BasicProc):
    """BasicProc + lattice_ids / lattice_lens [L * max_lattice_words] int32: for each character the vocabulary words of
    2..10 characters starting there (the giga tokenizer's characters, whitespace dropped), the most frequent
    max_lattice_words of them (NativeLexicon.build_lattice).  `word_embedding` (the [n_word + 3, Ew] table whose rows
    follow `vocab`) initialises the plugin's trainable word table.  `dropped` counts the matches the cap discarded."""

    def __init__(self, tokenizer_type, max_seq_len, tag2idx, tokenizer, vocab, word_embedding=None, vocabfreq=None,
                 max_lattice_words=MaxLatticeWords):
        _reject_bert(tokenizer_type, 'LatticeProc')
        super(LatticeProc, self).__init__(tokenizer_type, max_seq_len, tag2idx, tokenizer)
        self.vocab, self.word_embedding, self.max_lattice_words = vocab, word_embedding, int(max_lattice_words)
        self.word_enhance = 'lattice'
        self.lexicon = NativeLexicon(vocab, vocabfreq)
        self.dropped = 0

    def build_seq_features(self, sentences, n_threads=0):
        feats = [super(LatticeProc, self).build_seq_feature(s) for s in sentences]
        chars = [[c for c in s if c.strip()] for s in sentences]
        ids, lens, dropped = self.lexicon.build_lattice(chars, self.max_seq_len, self.max_lattice_words, n_threads)
        self.dropped += dropped
        for f, i, n in zip(feats, ids, lens):
            f['lattice_ids'], f['lattice_lens'] = i.tolist(), n.tolist()
        return feats

    def build_seq_feature(self, sentence):
        return self.build_seq_features([sentence], n_threads=1)[0]

    def build_data_params(self, n_sample):
        params = super(LatticeProc, self).build_data_params(n_sample)
        params.update({'max_lattice_words': self.max_lattice_words, 'vocab2idx': self.vocab.vocab2idx,
                       'word_embedding': self.word_embedding})
        return params


def lattice_word_embedding(vectors, seed=1234):
    """[n_word + 3, Ew] float32 table for a WordVocab over `vectors` (TextVectors): the word vectors, then N(0, 1) rows for
    <None> and <eos> and a zero row for <PAD> (the id of empty lattice slots)."""
    rng = np.random.RandomState(seed)
    v = np.asarray(vectors.vectors, np.float32)
    extra = rng.normal(0, 1, size=(3, v.shape[1])).astype(np.float32)
    extra[1] = 0.0
    return np.vstack([v, extra]).astype(np.float32)


def softword_labels(words):
    """Segmented words -> one B/M/E/S id per character (SoftWordIds)."""
    out = []
    for w in words:
        n = len(w)
        out += [SoftWordIds['S']] if n == 1 else [SoftWordIds['B']] + [SoftWordIds['M']] * (n - 2) + [SoftWordIds['E']]
    return out


class SoftWordProc(BasicProc):
    """BasicProc + softword_ids [L] int32: the B/M/E/S label (SoftWordIds) a word segmenter gives each character.
    `cut(sentence) -> iterable of words` segments the whitespace-stripped sentence; without one, jieba.cut is used when
    jieba is installed."""

    def __init__(self, tokenizer_type, max_seq_len, tag2idx, tokenizer, cut=None):
        _reject_bert(tokenizer_type, 'SoftWordProc')
        super(SoftWordProc, self).__init__(tokenizer_type, max_seq_len, tag2idx, tokenizer)
        if cut is None:
            try:
                import jieba
            except ImportError:
                raise ImportError('SoftWordProc needs a word segmenter: pass cut=<sentence -> words> or install jieba')
            cut = jieba.cut
        self.cut, self.word_enhance = cut, 'softword'

    def build_seq_feature(self, sentence):
        f = super(SoftWordProc, self).build_seq_feature(sentence)
        text = ''.join(c for c in sentence if c.strip())
        words = [w for w in self.cut(text) if w]
        if sum(len(w) for w in words) != len(text):
            raise ValueError('segmenter output does not cover the sentence {}...'.format(text[:10]))
        labels = softword_labels(words)[:self.max_seq_len]
        f['softword_ids'] = labels + [0] * (self.max_seq_len - len(labels))
        return f
