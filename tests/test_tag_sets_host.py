"""CPU: tag sets read from the data (preprocess --tag_set data / --tag_scheme bioes), their refusals, and the class table
of the GPU span extractor past 32 entity types."""
import os

import pytest

from chinesener_b200 import ops
from chinesener_b200.data import base_preprocess as bp
from chinesener_b200.data import preprocess as pp
from chinesener_b200.data.records import RecordFile
from chinesener_b200.data.tokenizer import TokenizerGiga
from chinesener_b200.tools.infer_utils import extract_entity


class _CharTok(object):
    def tokenize(self, s):
        return s.split(' ')

    def convert_tokens_to_ids(self, toks):
        return [0 if t == '[PAD]' else 1 + (ord(t[0]) % 50) for t in toks]


def _split(tmp_path, per_split):
    src = tmp_path / 'src'
    for name, (sents, tags) in per_split.items():
        d = src / name
        d.mkdir(parents=True, exist_ok=True)
        (d / 'sentences.txt').write_text('\n'.join(sents) + '\n', encoding='utf-8')
        (d / 'tags.txt').write_text('\n'.join(tags) + '\n', encoding='utf-8')
    return str(src)


def _dump(tmp_path, src, out, t2i, load=None):
    p = bp.BasicProc(TokenizerGiga, 8, t2i, _CharTok())
    return {name: pp.dump_records(p, src, str(tmp_path / out), name, verbose=False, load_data=load)
            for name in ('train', 'val', 'test')}


MSRA_SPLIT = (['a b c', 'd e', 'f'], ['B-PER I-PER O', 'O B-ORG', 'B-LOC'])


def test_msra_tag_set_is_byte_identical_to_the_default(tmp_path):
    src = _split(tmp_path, {n: MSRA_SPLIT for n in ('train', 'val', 'test')})
    _dump(tmp_path, src, 'default', pp.MSRA_TAG2IDX)
    _dump(tmp_path, src, 'msra', pp.MSRA_TAG2IDX, load=pp.scheme_loader('bio'))
    names = sorted(os.listdir(tmp_path / 'default'))
    assert names and names == sorted(os.listdir(tmp_path / 'msra'))
    for f in names:
        assert (tmp_path / 'default' / f).read_bytes() == (tmp_path / 'msra' / f).read_bytes(), f


def test_data_tag_set_order_and_data_params(tmp_path):
    t2i = pp.data_tag2idx(['B-PER I-PER O', 'B-GPE O B-ORG', 'O', 'B-FAC|O ?'])
    assert list(t2i) == ['[PAD]', 'O', 'B-FAC', 'I-FAC', 'B-GPE', 'I-GPE', 'B-ORG', 'I-ORG', 'B-PER', 'I-PER',
                         '[CLS]', '[SEP]']
    assert list(t2i.values()) == list(range(12))
    assert pp.data_tag2idx(['B-ORG I-ORG', 'B-PER I-PER O B-LOC I-LOC']) == {
        '[PAD]': 0, 'O': 1, 'B-LOC': 2, 'I-LOC': 3, 'B-ORG': 4, 'I-ORG': 5, 'B-PER': 6, 'I-PER': 7, '[CLS]': 8, '[SEP]': 9}
    params = bp.BasicProc(TokenizerGiga, 8, t2i, _CharTok()).build_data_params(3)
    assert params['label_size'] == 12 and params['tag2idx'] == t2i
    assert params['idx2tag'] == {v: k for k, v in t2i.items()}


def test_unknown_type_in_a_later_split_is_counted_invalid(tmp_path):
    train = (['a b', 'c'], ['B-AAA I-AAA', 'B-BBB'])
    val = (['a b', 'c', 'd'], ['B-AAA O', 'B-ZZZ', 'B-BBB'])
    src = _split(tmp_path, {'train': train, 'val': val, 'test': train})
    t2i = pp.data_tag2idx(pp.load_data(src, 'train')[1])
    n = _dump(tmp_path, src, 'out', t2i)
    assert n['train'] == (2, 0) and n['val'] == (2, 1)


def test_bioes_rewrites_to_bio_with_the_same_entities():
    toks = list('abcdefghijk')
    bioes = 'S-PER B-ORG M-ORG E-ORG O B-LOC E-LOC S-LOC O S-PER B-ORG'
    bio = pp.bioes_to_bio(bioes)
    assert bio == 'B-PER B-ORG I-ORG I-ORG O B-LOC I-LOC B-LOC O B-PER B-ORG'
    t2i = pp.data_tag2idx([bio])
    idx2tag = {v: k for k, v in t2i.items()}
    ids = [t2i[t] for t in bio.split(' ')]
    ents = extract_entity(toks, ids, idx2tag)
    assert ents == {'PER': {'a', 'j'}, 'ORG': {'bcd', 'k'}, 'LOC': {'fg', 'h'}}
    assert pp.bioes_to_bio('E-PER|S-LOC ? O') == 'I-PER|B-LOC ? O'


def test_bioes_loader_feeds_dump_records(tmp_path):
    split = (['a b c', 'd e'], ['B-PER M-PER E-PER', 'S-ORG O'])
    src = _split(tmp_path, {n: split for n in ('train', 'val', 'test')})
    load = pp.scheme_loader('bioes')
    t2i = pp.data_tag2idx(load(src, 'train')[1])
    n = _dump(tmp_path, src, 'out', t2i, load=load)
    assert n['train'] == (2, 0)
    b = RecordFile(str(tmp_path / 'out' / 'giga_train.nerrec')).batch(slice(0, 2))
    assert b['label_ids'][0].tolist()[:3] == [t2i['B-PER'], t2i['I-PER'], t2i['I-PER']]


def _types(n):
    return ['T%03d' % i for i in range(n)]


def test_more_than_128_tags_is_refused(tmp_path):
    ok = pp.data_tag2idx([' '.join('B-' + t for t in _types(62))])
    assert len(ok) == 128                                        # 62 types: the most a 128-tag BIO set holds
    with pytest.raises(ValueError, match="at most 128 tags"):
        pp.data_tag2idx([' '.join('B-' + t for t in _types(63))])
    src = _split(tmp_path, {n: (['a'] * 63, ['B-' + t for t in _types(63)]) for n in ('train', 'val', 'test')})
    with pytest.raises(ValueError, match="at most 128 tags"):
        pp.main(['--src', src, '--out', str(tmp_path / 'o'), '--tag_set', 'data', '--giga_vec', '/nonexistent'])


def test_partial_labels_past_32_tags_are_refused(tmp_path, capsys):
    src = _split(tmp_path, {n: (['a'] * 16, ['B-' + t for t in _types(16)]) for n in ('train', 'val', 'test')})
    with pytest.raises(SystemExit):
        pp.main(['--src', src, '--out', str(tmp_path / 'o'), '--tag_set', 'data', '--partial_labels',
                 '--giga_vec', '/nonexistent'])
    assert 'at most 32 tags' in capsys.readouterr().err
    with pytest.raises(SystemExit):
        pp.main(['--src', src, '--out', str(tmp_path / 'o'), '--format', 'msr', '--tag_set', 'data'])


def test_tag_classes_for_63_types():
    tags = ['[PAD]', 'O'] + [p + '-' + t for t in _types(63) for p in ('B', 'I')] + ['[CLS]', '[SEP]']
    idx2tag = dict(enumerate(tags))
    table, types = ops.tag_classes(idx2tag)
    assert table.dtype.itemsize == 2 and len(types) == 63
    for i, tag in idx2tag.items():
        v = int(table[i])
        if tag[:2] in ('B-', 'I-'):
            assert v & 3 == (1 if tag[0] == 'B' else 2) and v & 4 and types[v >> 3] == tag[2:]
        else:
            assert v == 0
    narrow, types32 = ops.tag_classes({v: k for k, v in pp.data_tag2idx([' '.join('B-' + t for t in _types(32))]).items()})
    assert narrow.dtype.itemsize == 1 and len(types32) == 32
