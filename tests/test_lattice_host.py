# -*-coding:utf-8 -*-
"""CPU: the native lattice lists (ner_lexicon_build_lattice) against the Python restatement in tests/_lattice_oracle.py, the
.nerrec round trip of the new columns, `preprocess --word_enhance lattice`, and the plugin-name mapping."""
import os
import pickle

import numpy as np
import pytest

from chinesener_b200.data import base_preprocess as bp, preprocess, records
from chinesener_b200.data.tokenizer import TokenizerAdapter, TokenizerBert, TokenizerGiga
from chinesener_b200.data.word_enhance import LatticeProc, NativeLexicon, WordVocab
from chinesener_b200.inference import TAG2IDX

import _lattice_oracle as olat
from test_dataset_pipeline import SAMPLE, _sample_dir
from test_word_enhance_host import write_vec


def _random_case(seed, n_sent=60, alphabet='甲乙丙丁戊己庚辛'):
    rng = np.random.default_rng(seed)
    sents = [''.join(rng.choice(list(alphabet), int(rng.integers(0, 40)))) for _ in range(n_sent)]
    sents[0] = ''                                                           # empty row
    sents[1] = alphabet * 3                                                  # long matches everywhere
    words = {sents[1][i:i + n] for n in range(2, 11) for i in range(0, 4)}     # > Kw words per start: the cap bites
    for s in sents[2:]:
        for _ in range(6):
            if len(s) >= 2:
                n = int(rng.integers(2, min(10, len(s)) + 1))
                i = int(rng.integers(0, len(s) - n + 1))
                words.add(s[i:i + n])
    words.update([alphabet[:10] if len(alphabet) >= 10 else alphabet, alphabet[:2], alphabet[0]])   # 1 char: never a lattice word
    words = sorted(words)
    counts = {w: int(rng.integers(1, 4)) for w in words}                   # few distinct counts: ties are frequent
    return sents, WordVocab(words, counts)


@pytest.mark.parametrize("seed,L,Kw", [(0, 32, 4), (1, 16, 2), (2, 48, 8), (3, 20, 1)])
def test_native_lattice_lists_match_the_restatement(seed, L, Kw):
    sents, vocab = _random_case(seed)
    ids, lens, dropped = NativeLexicon(vocab).build_lattice([list(s) for s in sents], L, Kw, n_threads=3)
    want_dropped = 0
    for s, i, n in zip(sents, ids, lens):
        ri, rn, rd = olat.lattice_words(list(s), vocab, L, Kw)
        assert i.tolist() == ri and n.tolist() == rn, s
        want_dropped += rd
    assert dropped == want_dropped and dropped > 0           # the cap bites on this vocabulary
    assert (lens[0] == 0).all() and (ids[0] == vocab.vocab2idx['<PAD>']).all()
    assert lens.max() <= 10 and (lens[lens > 0] >= 2).all()


def test_max_length_words_and_tie_order():
    vocab = WordVocab(['一二三四五六七八九十', '一二', '一二三', '二三'], {'一二三四五六七八九十': 1, '一二': 1, '一二三': 2, '二三': 1})
    ids, lens, dropped = NativeLexicon(vocab).build_lattice([list('一二三四五六七八九十')], 12, 2)
    # start 0 matches 一二 (1), 一二三 (2), 10 characters (1): the cap keeps 一二三 then the first of the tied pair
    assert lens[0][:2].tolist() == [3, 2] and ids[0][:2].tolist() == [2, 1] and dropped == 1
    ids, lens, _ = NativeLexicon(vocab).build_lattice([list('一二三四五六七八九十')], 12, 4)
    assert lens[0][:4].tolist() == [2, 3, 10, 0]             # trie order: increasing length
    ids, lens, _ = NativeLexicon(vocab).build_lattice([list('一二三四五六七八九十')], 9, 4)
    assert lens[0][:4].tolist() == [2, 3, 0, 0]              # the 10-character word ends past max_seq_len


def test_model_name_mapping_and_bert_refusal():
    assert bp.extract_prefix_surfix('lattice_lstm_crf') == ('lattice', TokenizerGiga)
    for name, want in (('bilstm_crf_softlexicon', 'softlexicon'), ('bilstm_crf_ex_softword', 'ex_softword'),
                       ('bilstm_crf_bichar', 'bichar'), ('bert_crf', None)):
        assert bp.extract_prefix_surfix(name)[0] == want
    tok = TokenizerAdapter(list('中国人'))
    vocab = WordVocab(['中国'], {'中国': 1})
    proc = bp.get_instance(TokenizerGiga, 8, TAG2IDX, tok, word_enhance='lattice', vocab=vocab,
                           word_embedding=np.zeros((4, 3), np.float32))
    assert type(proc) is LatticeProc
    f = proc.build_seq_feature('中 国人')
    assert f['lattice_lens'][:4] == [2, 0, 0, 0] and f['lattice_ids'][:2] == [0, 2]
    batch = bp.features_to_batch([f])
    assert batch['lattice_ids'].shape == (1, 32) and batch['lattice_lens'].shape == (1, 32)
    p = proc.build_data_params(1)
    assert p['max_lattice_words'] == 4 and p['word_embedding'].shape == (4, 3) and p['vocab2idx'] is vocab.vocab2idx
    with pytest.raises(ValueError, match='BERT'):
        bp.get_instance(TokenizerBert, 8, TAG2IDX, tok, word_enhance='lattice', vocab=vocab)


def test_nerrec_round_trip_of_the_lattice_columns(tmp_path):
    sents, vocab = _random_case(5, n_sent=9)
    sents = [s for s in sents if s]
    tok = TokenizerAdapter(sorted(set(''.join(sents))))
    proc = LatticeProc(TokenizerGiga, 24, TAG2IDX, tok, vocab)
    feats = proc.build_seq_features(sents)
    for f in feats:
        f.update(proc.build_tag_feature(' '.join(['O'] * f['seq_len'])))
    path = str(tmp_path / 'x.nerrec')
    records.write_records(path, feats, 24)
    rf = records.RecordFile(path)
    b = rf.batch(np.arange(len(feats)), with_strings=False)
    for k in ('lattice_ids', 'lattice_lens'):
        assert b[k].dtype == records.torch.int32
        np.testing.assert_array_equal(b[k].numpy(), np.asarray([f[k] for f in feats]))


def test_preprocess_lattice_cli_round_trips_through_nerdataset(tmp_path):
    src = _sample_dir(tmp_path)
    giga = write_vec(tmp_path / 'giga.vec', SAMPLE['giga_vocab_subset'], dim=50)
    text = [s.replace(' ', '') for s in SAMPLE['sentences']]
    words = sorted({t[i:i + n] for t in text for n in (2, 3, 4) for i in range(0, len(t) - n, 3)})
    preprocess.main(['--src', src, '--out', str(tmp_path / 'out'), '--tokenizer', 'giga', '--giga_vec', giga,
                     '--word_enhance', 'lattice', '--word_vec', write_vec(tmp_path / 'word.vec', words, dim=16, seed=2)])
    out = str(tmp_path / 'out')
    assert sorted(os.listdir(out)) == sorted(['giga_{}_lattice.nerrec'.format(s) for s in ('train', 'valid', 'predict')]
                                             + ['giga_lattice_data_params.pkl'])
    params = pickle.load(open(os.path.join(out, 'giga_lattice_data_params.pkl'), 'rb'))
    assert params['max_lattice_words'] == 4 and params['word_embedding'].shape == (len(words) + 3, 16)
    assert (params['word_embedding'][len(words) + 1] == 0).all()              # <PAD>: the id of empty slots
    ds = records.NerDataset(out, batch_size=5, epoch_size=1, model_name='lattice_lstm_crf')
    b = next(iter(ds.build_input_fn('predict', is_predict=True)()))
    assert b['lattice_ids'].shape == b['lattice_lens'].shape == (5, 150 * 4)
    assert b['lattice_lens'].max() >= 2
    # the stored lists are what the processor builds for the same sentences
    vocab = WordVocab(words, dict.fromkeys(words, 1))
    lens = NativeLexicon(vocab).build_lattice([[c for c in s if c.strip()] for s in SAMPLE['sentences']], 150)[1]
    assert any((np.asarray(b['lattice_lens'][i]) == lens[j]).all() for i in range(5) for j in range(len(lens)))
