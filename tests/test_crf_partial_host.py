"""CPU: partial labels in the data path: '?' / 'T1|T2' parsing in BasicProc.build_tag_feature, the label_mask rows,
rejection of bad sets, the .nerrec round trip of label_mask (bit 31 included), files byte-identical to the ordinary
ones when no position is open, the batch dict, and SingleEval's refusal of partial labels."""
import os

import numpy as np
import pytest

from chinesener_b200.data import base_preprocess as bp
from chinesener_b200.data import preprocess as pp
from chinesener_b200.data.records import RecordFile, write_records
from chinesener_b200.data.tokenizer import TokenizerBert, TokenizerGiga
from chinesener_b200.evaluation import SingleEval

T2I = pp.MSRA_TAG2IDX                      # [PAD] 0, O 1, B-ORG 2, ..., I-LOC 7, [CLS] 8, [SEP] 9
REAL = sum(1 << i for t, i in T2I.items() if t not in ('[PAD]', '[CLS]', '[SEP]'))


class _CharTok(object):
    def tokenize(self, s):
        return s.split(' ')

    def convert_tokens_to_ids(self, toks):
        return [0 if t == '[PAD]' else 1 + (ord(t[0]) % 50) for t in toks]


def _proc(kind=TokenizerGiga, L=8, partial=True):
    p = bp.BasicProc(kind, L, T2I, _CharTok())
    p.partial_labels = partial
    return p


def test_open_and_set_tags_giga():
    f = _proc().build_tag_feature('B-PER ? I-LOC|O O')
    assert f['label_ids'] == [4, -1, -1, 1, 0, 0, 0, 0]
    assert f['label_mask'] == [1 << 4, REAL, (1 << 7) | (1 << 1), 1 << 1, 1, 1, 1, 1]     # [PAD]: its one-hot bit
    assert f['labels'][:4] == ['B-PER', '?', 'I-LOC|O', 'O'] and f['label_len'] == 4


def test_cls_sep_get_their_exact_bit():
    f = _proc(TokenizerBert).build_tag_feature('? O')
    assert f['label_ids'][:4] == [8, -1, 1, 9]
    assert f['label_mask'][:5] == [1 << 8, REAL, 1 << 1, 1 << 9, 1]


@pytest.mark.parametrize("bad", ['B-PER|FOO', '[CLS]|O', 'O|[PAD]', 'B-PER|', '??'])
def test_bad_sets_are_rejected(bad):
    with pytest.raises((ValueError, KeyError)):
        _proc().build_tag_feature('O ' + bad)


def test_without_the_flag_open_tags_are_unknown_tags():
    with pytest.raises(KeyError):
        _proc(partial=False).build_tag_feature('O ?')
    assert 'label_mask' not in _proc(partial=False).build_tag_feature('O B-PER')


def test_bit_31_is_the_sign_bit():
    t2i = {'[PAD]': 0, **{'T%d' % i: i for i in range(1, 32)}}
    p = bp.BasicProc(TokenizerGiga, 3, t2i, _CharTok())
    p.partial_labels = True
    f = p.build_tag_feature('T31|T1 ?')
    assert f['label_mask'][0] == -(1 << 31) | 2
    assert f['label_mask'][1] == -2                                # bits 1..31
    assert f['label_mask'][2] == 1


def test_nerrec_round_trip_of_label_mask(tmp_path):
    t2i = {'[PAD]': 0, **{'T%d' % i: i for i in range(1, 32)}}
    p = bp.BasicProc(TokenizerGiga, 4, t2i, _CharTok())
    p.partial_labels = True
    feats = [p.build_feature('a b c', 'T31 ? T2|T31'), p.build_feature('d e', 'T1 T5')]
    path = str(tmp_path / 'x.nerrec')
    write_records(path, feats, 4)
    batch = RecordFile(path).batch(slice(0, 2))
    assert batch['label_mask'].tolist() == [f['label_mask'] for f in feats]
    assert batch['label_ids'].tolist() == [[31, -1, -1, 0], [1, 5, 0, 0]]
    host = bp.features_to_batch(feats)
    assert host['label_mask'].tolist() == batch['label_mask'].tolist()


def _split(tmp_path, tags):
    src = tmp_path / 'src'
    for name in ('train', 'val', 'test'):
        d = src / name
        d.mkdir(parents=True, exist_ok=True)
        (d / 'sentences.txt').write_text('\n'.join(['a b c', 'd e', 'f'] * 2) + '\n', encoding='utf-8')
        (d / 'tags.txt').write_text('\n'.join(tags * 2) + '\n', encoding='utf-8')
    return str(src)


def _dump(tmp_path, src, out, partial):
    p = _proc(L=6, partial=partial)
    n = {}
    for name in ('train', 'val', 'test'):
        n[name] = pp.dump_records(p, src, str(tmp_path / out), name, verbose=False)
    return n


def test_fully_labelled_files_are_byte_identical(tmp_path):
    src = _split(tmp_path, ['B-PER I-PER O', 'O O', 'B-LOC'])
    _dump(tmp_path, src, 'plain', False)
    _dump(tmp_path, src, 'flag', True)
    for f in sorted(os.listdir(tmp_path / 'plain')):
        assert (tmp_path / 'plain' / f).read_bytes() == (tmp_path / 'flag' / f).read_bytes(), f


def test_partial_split_gets_the_column_and_bad_sets_count_as_invalid(tmp_path):
    src = _split(tmp_path, ['B-PER ? O', 'O B-FOO|O', 'B-LOC'])
    n = _dump(tmp_path, src, 'out', True)
    assert n['train'] == (4, 2)                               # the 'B-FOO|O' sentences are dropped and counted
    rec = RecordFile(str(tmp_path / 'out' / 'giga_train.nerrec'))
    assert 'label_mask' in rec.names()
    b = rec.batch(slice(0, 4))
    assert b['label_ids'][0].tolist()[:3] == [4, -1, 1]
    assert b['label_mask'][0].tolist()[:4] == [1 << 4, REAL, 1 << 1, 1]
    assert b['label_mask'][1].tolist()[:2] == [1 << 6, 1]     # a fully labelled sentence of the split: one-hot rows


def test_single_eval_refuses_partial_labels():
    idx2tag = {v: k for k, v in T2I.items()}
    pred = [{'pred_ids': np.array([1, 1, 0], np.int32), 'label_ids': np.array([1, -1, 0], np.int32),
             'tokens': np.array([b'a', b'b', b'[PAD]'], dtype=object)}]
    with pytest.raises(ValueError, match='partial labels'):
        SingleEval(pred, idx2tag)
