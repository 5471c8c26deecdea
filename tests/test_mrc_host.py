# -*-coding:utf-8 -*-
"""Host side of the bert_mrc plugin (no GPU): entity types and queries (data/mrc.py), and the numpy restatement of its
kernels (tests/_mrc_oracle.py) pinned by hand-worked examples."""
import json

import numpy as np
import pytest

from _mrc_oracle import mrc_merge, mrc_pairs
from chinesener_b200.data import mrc
from chinesener_b200.data.preprocess import MSRA_TAG2IDX

MSRA_IDX2TAG = {i: t for t, i in MSRA_TAG2IDX.items()}


def _pretrain_dir(tmp_path, max_position=512, vocab=None):
    (tmp_path / "bert_config.json").write_text(json.dumps({'vocab_size': 200, 'max_position_embeddings': max_position}))
    if vocab is not None:
        (tmp_path / "vocab.txt").write_text("\n".join(vocab) + "\n", encoding="utf-8")
    return str(tmp_path)


def _params(pretrain_dir, L=128, idx2tag=MSRA_IDX2TAG, **extra):
    return dict(idx2tag=idx2tag, max_seq_len=L, pretrain_dir=pretrain_dir, **extra)


def test_entity_types_follow_the_tag_ids():
    assert mrc.entity_types(MSRA_IDX2TAG) == [('ORG', 2, 3), ('PER', 4, 5), ('LOC', 6, 7)]
    swapped = {0: 'O', 1: 'B-LOC', 2: 'I-LOC', 3: 'B-PER', 4: 'I-PER'}
    assert [n for n, _, _ in mrc.entity_types(swapped)] == ['LOC', 'PER']


def test_queries_are_tokenized_with_the_bert_vocabulary(tmp_path):
    chars = sorted(set(''.join(mrc.DEFAULT_QUERIES.values())))
    vocab = ['[PAD]', '[UNK]', '[CLS]', '[SEP]'] + chars
    table = mrc.MrcTable(_params(_pretrain_dir(tmp_path, vocab=vocab)), device='cpu')
    assert table.names == ['ORG', 'PER', 'LOC'] and table.T == 3
    assert table.query_lens == [22, 10, 20]                         # one token per character and comma
    assert table.qmax == 22 and table.L2 == 22 + 1 + 128
    assert table.query_overhead == 52 + 3
    assert table.sep_id == 3
    idx = {c: i for i, c in enumerate(vocab)}
    for t, name in enumerate(table.names):
        q = mrc.DEFAULT_QUERIES[name]
        assert table.query_ids[t, :len(q)].tolist() == [idx[c] for c in q]
        assert not table.query_ids[t, len(q):].any()
    assert table.type_tag.tolist() == [[2, 3], [4, 5], [6, 7]]
    assert (table.o_tag, table.cls_tag, table.sep_tag) == (1, 8, 9)
    # host pair token count: T * tokens + (q_t + 1 summed over types) * non-empty sentences
    mask = np.zeros((3, 128), np.int32)
    mask[0, :5], mask[2, :128] = 1, 1

    class Mask:
        total_tokens, nonempty_rows = int(mask.sum()), 2
    assert table.pair_tokens(Mask) == 3 * 133 + 55 * 2
    assert table.pair_tokens(object()) is None


def test_query_ids_override_and_custom_queries(tmp_path):
    table = mrc.MrcTable(_params('', L=16, mrc_query_ids={'ORG': [7, 8], 'PER': [], 'LOC': [9]}), device='cpu')
    assert table.query_lens == [2, 0, 1] and table.qmax == 2 and table.L2 == 19
    assert table.query_ids.tolist() == [[7, 8], [0, 0], [9, 0]]
    assert table.sep_id == mrc.SEP_TOKEN_ID                         # no vocabulary: BERT-Base-Chinese's [SEP]
    vocab = ['[PAD]', '[UNK]', '[CLS]', '[SEP]', '甲', '乙']
    queries = {'ORG': '甲乙', 'PER': '乙', 'LOC': '丙'}
    table = mrc.MrcTable(_params(_pretrain_dir(tmp_path, vocab=vocab), mrc_queries=queries), device='cpu')
    assert table.query_ids.tolist() == [[4, 5], [5, 0], [1, 0]]     # 丙 is not in the vocabulary: [UNK]
    # no [CLS] / [SEP] tags: both positions fall back to O
    plain = {0: '[PAD]', 1: 'O', 2: 'B-X', 3: 'I-X'}
    table = mrc.MrcTable(_params('', L=8, idx2tag=plain, mrc_query_ids={'X': [5]}), device='cpu')
    assert (table.o_tag, table.cls_tag, table.sep_tag) == (1, 1, 1)


def test_errors_name_the_problem(tmp_path):
    with pytest.raises(KeyError, match="'LOC'"):
        mrc.MrcTable(_params('', mrc_query_ids={'ORG': [1], 'PER': [2]}), device='cpu')
    vocab = ['[PAD]', '[UNK]', '[CLS]', '[SEP]']
    with pytest.raises(KeyError, match="'PER'"):
        mrc.MrcTable(_params(_pretrain_dir(tmp_path, vocab=vocab), mrc_queries={'ORG': 'a', 'LOC': 'b'}), device='cpu')
    with pytest.raises(ValueError, match="max_position_embeddings"):
        mrc.MrcTable(_params(_pretrain_dir(tmp_path, max_position=140), mrc_query_ids={'ORG': [1] * 12, 'PER': [2], 'LOC': [3]}),
                     device='cpu')
    # 12 + 1 + 128 = 141 > 140; one token shorter fits
    mrc.MrcTable(_params(_pretrain_dir(tmp_path, max_position=140), mrc_query_ids={'ORG': [1] * 11, 'PER': [2], 'LOC': [3]}),
                 device='cpu')
    many = {0: 'O'}
    for k in range(33):
        many[1 + 2 * k], many[2 + 2 * k] = f'B-T{k}', f'I-T{k}'
    with pytest.raises(ValueError, match="1 to 32"):
        mrc.MrcTable(_params('', idx2tag=many, mrc_query_ids={f'T{k}': [1] for k in range(33)}), device='cpu')
    with pytest.raises(ValueError, match="1 to 32"):
        mrc.entity_types({0: 'O', 1: '[CLS]'})
    with pytest.raises(ValueError, match="I-X"):
        mrc.entity_types({0: 'O', 1: 'B-X'})
    with pytest.raises(FileNotFoundError, match="mrc_query_ids"):         # no vocabulary and no query ids
        mrc.query_token_ids(dict(pretrain_dir=str(tmp_path / "absent")), ['ORG'])


# --------------------------------------------------------------------------- the oracle, by hand
def test_pairs_oracle_hand_worked():
    """L = 4, T = 2 with queries of 2 and 0 tokens (Qmax 2, L2 = 7); seq_len 0, 1, 2, 4."""
    token_ids = np.array([[0, 0, 0, 0], [101, 0, 0, 0], [101, 102, 0, 0], [101, 21, 22, 102]], np.int32)
    label_ids = np.array([[0, 0, 0, 0], [8, 0, 0, 0], [8, 9, 0, 0], [8, 4, 3, 9]], np.int32)
    out = mrc_pairs(token_ids, [0, 1, 2, 4], [[11, 12], [0, 0]], [2, 0], [[2, 3], [4, 5]], 7, 102, label_ids)
    assert out['ids'].tolist() == [
        [0, 0, 0, 0, 0, 0, 0], [0, 0, 0, 0, 0, 0, 0],                          # empty sentence: empty pairs
        [101, 11, 12, 102, 0, 0, 0], [101, 102, 0, 0, 0, 0, 0],                # [CLS] only: [CLS] q [SEP]
        [101, 11, 12, 102, 102, 0, 0], [101, 102, 102, 0, 0, 0, 0],
        [101, 11, 12, 102, 21, 22, 102], [101, 102, 21, 22, 102, 0, 0]]
    assert out['mask'].sum(1).tolist() == [0, 0, 4, 2, 5, 3, 7, 5]
    assert out['segment_ids'].tolist() == [
        [0] * 7, [0] * 7, [0] * 7, [0] * 7,
        [0, 0, 0, 0, 1, 0, 0], [0, 0, 1, 0, 0, 0, 0],
        [0, 0, 0, 0, 1, 1, 1], [0, 0, 1, 1, 1, 0, 0]]
    assert out['seq_len'].tolist() == [0, 0, 1, 1, 2, 2, 4, 4]
    assert out['align'].reshape(8, 4).tolist() == [
        [0, 4, 5, 6], [7, 9, 10, 11], [14, 18, 19, 20], [21, 23, 24, 25],
        [28, 32, 33, 34], [35, 37, 38, 39], [42, 46, 47, 48], [49, 51, 52, 53]]
    assert out['labels'].tolist() == [[0] * 4] * 6 + [[0, 0, 2, 0], [0, 1, 0, 0]]
    # every real sentence position reads its own token through the alignment
    flat = out['ids'].reshape(-1)
    for p in range(8):
        b, n = p // 2, out['seq_len'][p]
        assert (flat[out['align'].reshape(8, 4)[p, :n]] == token_ids[b, :n]).all()
    assert mrc_pairs(token_ids, [0, 1, 2, 4], [[11, 12], [0, 0]], [2, 0], [[2, 3], [4, 5]], 7, 102)['labels'] is None


def test_merge_oracle_hand_worked():
    """T = 2 (ORG, PER tags 2/3, 4/5), O = 1, [CLS] = 8, [SEP] = 9; seq_len 5, 0, 1, 2."""
    L = 5
    z = np.zeros((4 * 2, L, 3), np.float32)
    z[0, 1], z[1, 1] = [0, 2, 0], [0, 0, 3]       # both claim s = 1; PER's I has the higher score -> I-PER
    z[0, 2], z[1, 2] = [1, 0, 0], [5, 0, 0]       # nobody claims s = 2 -> O
    z[0, 3], z[1, 3] = [0, 1, 0], [0, 1, 0]       # tie -> the lower type index, B-ORG
    z[2:] = np.random.default_rng(0).normal(size=(6, L, 3)) * 3
    pred, margin = mrc_merge(z, [5, 0, 1, 2], [[2, 3], [4, 5]], 1, 8, 9)
    assert pred.tolist() == [[8, 5, 1, 2, 9], [0] * 5, [8, 0, 0, 0, 0], [8, 9, 0, 0, 0]]
    s_org, s_per = -np.log(1 + 2 * np.exp(-2)), -np.log(1 + 2 * np.exp(-3))
    assert abs(margin[0, 1] - min(s_per - s_org, 2.0)) < 1e-6
    assert margin[0, 3] == 0.0 and np.isinf(margin[0, 0]) and np.isinf(margin[1]).all()
