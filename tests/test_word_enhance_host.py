# -*-coding:utf-8 -*-
"""CPU: host featurisation of the word-enhance plugins (BiCharProc, ExSoftWordProc, SoftWordProc), get_instance, and
`preprocess --word_enhance ...` read back through NerDataset."""
import os
import pickle

import numpy as np
import pytest

from chinesener_b200.data import base_preprocess as bp, preprocess, records
from chinesener_b200.data.tokenizer import TokenizerAdapter, TokenizerBert, TokenizerGiga
from chinesener_b200.data.word_enhance import (BiCharProc, ExSoftWordProc, SoftWordProc, WordVocab, giga_chars,
                                               softword_labels)
from chinesener_b200.inference import TAG2IDX

from test_dataset_pipeline import SAMPLE, _sample_dir


def test_bichar_ids_on_a_hand_worked_sentence():
    chars = TokenizerAdapter(['A', 'B', '中', '文'])
    bichars = TokenizerAdapter(['AB', 'B中', '文-null-'])          # [PAD] = 3, [UNK] = 4
    proc = BiCharProc(TokenizerGiga, 6, TAG2IDX, chars, bichars)
    f = proc.build_seq_feature('ＡB中 文')                         # full-width A folds to A, the space is dropped
    assert f['tokens'][:4] == ['A', 'B', '中', '文'] and f['seq_len'] == 4
    # AB, B中, 中文 (out of vocabulary), 文 + end marker, then [PAD]
    assert f['bichar_ids'] == [0, 1, 4, 2, 3, 3]
    short = BiCharProc(TokenizerGiga, 3, TAG2IDX, chars, bichars).build_seq_feature('ＡB中 文')
    assert short['bichar_ids'] == [0, 1, 4]                       # truncated: position 2 still pairs with its real neighbour


def _brute_force_ex_softword(sentence, words, L):
    text = sentence.replace(' ', '')
    out = np.zeros((L, 5), np.float32)
    sets = [set() for _ in text]
    for i in range(len(text)):
        for j in range(i, min(i + 10, len(text))):
            if text[i:j + 1] in words:
                if i == j:
                    sets[i].add(3)
                else:
                    sets[i].add(0)
                    sets[j].add(2)
                    for k in range(i + 1, j):
                        sets[k].add(1)
    for r in range(min(len(text), L)):
        for g in sets[r]:
            out[r, g] = 1
        out[r, 4] = 0 if sets[r] else 1
    return out.reshape(-1)


def test_ex_softword_against_a_brute_force_substring_scan():
    rng = np.random.default_rng(0)
    alphabet = list('甲乙丙丁戊己庚')
    words = sorted({''.join(rng.choice(alphabet, n)) for n in rng.integers(1, 5, 40)})
    vocab = WordVocab(words, dict.fromkeys(words, 1))
    L = 24
    proc = ExSoftWordProc(TokenizerGiga, L, TAG2IDX, TokenizerAdapter(alphabet), vocab)
    sents = [''.join(rng.choice(alphabet, n)) for n in rng.integers(0, 40, 60)] + ['甲 乙丙']
    feats = proc.build_seq_features(sents)
    for s, f in zip(sents, feats):
        np.testing.assert_array_equal(np.asarray(f['ex_softword_ids'], np.float32), _brute_force_ex_softword(s, set(words), L), s)
    assert proc.build_seq_feature(sents[3])['ex_softword_ids'] == feats[3]['ex_softword_ids']


def test_softword_labels_from_an_injected_segmenter():
    assert softword_labels(['我', '爱北京', '天安门', '了']) == [4, 1, 2, 3, 1, 2, 3, 4]
    cuts = []

    def cut(text):
        cuts.append(text)
        return ['我', '爱', '北京', '天安门']
    proc = SoftWordProc(TokenizerGiga, 10, TAG2IDX, TokenizerAdapter(list('我爱北京天安门')), cut=cut)
    f = proc.build_seq_feature('我爱 北京天安门')
    assert cuts == ['我爱北京天安门']                               # segments the whitespace-stripped sentence
    assert f['softword_ids'] == [4, 4, 1, 3, 1, 2, 3, 0, 0, 0] and f['seq_len'] == 7
    assert SoftWordProc(TokenizerGiga, 4, TAG2IDX, proc.tokenizer, cut=cut).build_seq_feature('我爱北京天安门')['softword_ids'] == [4, 4, 1, 3]
    with pytest.raises(ValueError):
        SoftWordProc(TokenizerGiga, 10, TAG2IDX, proc.tokenizer, cut=lambda s: ['我']).build_seq_feature('我爱北京')


def test_softword_without_a_segmenter_names_the_missing_one():
    try:
        import jieba  # noqa: F401
        pytest.skip('jieba is installed')
    except ImportError:
        pass
    with pytest.raises(ImportError, match='jieba'):
        SoftWordProc(TokenizerGiga, 10, TAG2IDX, TokenizerAdapter(['a']))


def test_get_instance_builds_all_three_and_rejects_bert():
    tok = TokenizerAdapter(list('中国人'))
    vocab = WordVocab(['中国'], {'中国': 1})
    kw = {'bichar': dict(bichar_tokenizer=TokenizerAdapter(['中国'])), 'softword': dict(cut=lambda s: [s]),
          'ex_softword': dict(vocab=vocab)}
    cls = {'bichar': BiCharProc, 'softword': SoftWordProc, 'ex_softword': ExSoftWordProc}
    col = {'bichar': 'bichar_ids', 'softword': 'softword_ids', 'ex_softword': 'ex_softword_ids'}
    for name, k in kw.items():
        proc = bp.get_instance(TokenizerGiga, 8, TAG2IDX, tok, word_enhance=name, **k)
        assert type(proc) is cls[name]
        f = proc.build_seq_feature('中国人')
        batch = bp.features_to_batch([f])
        assert batch[col[name]].shape == (1, 8 * (5 if name == 'ex_softword' else 1))
        with pytest.raises(ValueError, match='BERT'):
            bp.get_instance(TokenizerBert, 8, TAG2IDX, tok, word_enhance=name, **k)
    assert giga_chars('Ａ b　c') == ['A', 'b', 'c']


def write_vec(path, words, dim=8, seed=0):
    rng = np.random.default_rng(seed)
    with open(path, 'w', encoding='utf-8') as f:
        for w in words:
            f.write(w + ' ' + ' '.join('%.5f' % x for x in rng.normal(size=dim)) + '\n')
    return str(path)


def prepare_corpus(tmp_path, word_enhance):
    """The MSRA sample as raw splits + giga / bigram / word vectors -> `preprocess --word_enhance` output dir."""
    src = _sample_dir(tmp_path)
    giga = write_vec(tmp_path / 'giga.vec', SAMPLE['giga_vocab_subset'], dim=50)
    text = [s.replace(' ', '') for s in SAMPLE['sentences']]
    grams = sorted({t[i:i + 2] for t in text for i in range(0, len(t) - 1, 3)})
    words = sorted({t[i:i + n] for t in text for n in (2, 3) for i in range(0, len(t) - n, 5)})
    args = ['--src', src, '--out', str(tmp_path / 'out'), '--tokenizer', 'giga', '--giga_vec', giga,
            '--word_enhance', word_enhance]
    if word_enhance == 'bichar':
        args += ['--bichar_vec', write_vec(tmp_path / 'bi.vec', grams, dim=50, seed=1)]
    if word_enhance == 'ex_softword':
        args += ['--word_vec', write_vec(tmp_path / 'word.vec', words, seed=2)]
    preprocess.main(args)
    return str(tmp_path / 'out')


@pytest.mark.parametrize('word_enhance', ['bichar', 'ex_softword'])
def test_preprocess_word_enhance_cli_round_trips_through_nerdataset(tmp_path, word_enhance):
    out = prepare_corpus(tmp_path, word_enhance)
    assert sorted(os.listdir(out)) == sorted(['giga_{}_{}.nerrec'.format(s, word_enhance) for s in ('train', 'valid', 'predict')]
                                             + ['giga_{}_data_params.pkl'.format(word_enhance)])
    ds = records.NerDataset(out, batch_size=5, epoch_size=1, model_name='bilstm_crf_' + word_enhance)
    assert ds.params['n_sample'] == 16 and ds.params['embedding'].shape[1] == 50
    assert ('bichar_embedding' in ds.params) == (word_enhance == 'bichar')
    b = next(iter(ds.build_input_fn('predict', is_predict=True)()))
    L = ds.params['max_seq_len']
    if word_enhance == 'bichar':
        ids = b['bichar_ids']
        assert ids.shape == (5, L) and int(ids.max()) < ds.params['bichar_embedding'].shape[0]
        pad = ds.params['bichar_embedding'].shape[0] - 2
        assert all((ids[i, n:] == pad).all() and (ids[i, :n] != pad).all() for i, n in enumerate(b['seq_len'].tolist()))
    else:
        x = b['ex_softword_ids'].view(5, L, 5)
        live = np.arange(L)[None, :] < b['seq_len'].numpy()[:, None]
        assert (x.sum(-1).numpy()[live] >= 1).all() and (x.numpy()[~live] == 0).all()
        assert x[..., :4].sum() > 0                                 # some characters matched a word


def test_softword_records_with_an_injected_segmenter(tmp_path):
    src = _sample_dir(tmp_path)
    tok = TokenizerAdapter(SAMPLE['giga_vocab_subset'])
    proc = bp.get_instance(TokenizerGiga, 150, preprocess.MSRA_TAG2IDX, tok, word_enhance='softword',
                           cut=lambda s: [s[i:i + 2] for i in range(0, len(s), 2)])
    out = str(tmp_path / 'out')
    for split in preprocess.MAPPING:
        preprocess.dump_records(proc, src, out, split, word_enhance='softword', verbose=False,
                                embedding=np.zeros((len(tok.vocab2idx), 50), np.float32))
    ds = records.NerDataset(out, batch_size=4, epoch_size=1, model_name='bilstm_crf_softword')
    b = next(iter(ds.build_input_fn('predict', is_predict=True)()))
    n = int(b['seq_len'][0])
    want = ([1, 3] * 200)[:n] if n % 2 == 0 else ([1, 3] * 200)[:n - 1] + [4]
    assert b['softword_ids'][0].tolist() == want + [0] * (150 - n)
    with open(os.path.join(out, 'giga_softword_data_params.pkl'), 'rb') as f:
        assert pickle.load(f)['n_sample'] == 16
