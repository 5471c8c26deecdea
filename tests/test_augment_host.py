"""CPU: the augmentation pools, the parsing and checks of the params, every refusal, and the invariants of the oracle's
rules on random rows."""
import json
import os
from collections import Counter

import numpy as np
import pytest

import _augment_oracle as ao
from chinesener_b200 import augment, engine
from chinesener_b200.data import records
from chinesener_b200.synthetic import MSRA_IDX2TAG

TAG2IDX = {v: k for k, v in MSRA_IDX2TAG.items()}     # [PAD] 0, O 1, B-ORG 2, I-ORG 3, B-PER 4, I-PER 5, B-LOC 6, I-LOC 7
PAD, O, BO, IO, BP, IP, BL, IL, CLS, SEP = range(10)


def _rows(bert):
    """Three hand-written rows: a two-token PER, a stray I-LOC, a one-token ORG and a three-token LOC."""
    rows = [([11, 12, 13, 14, 15], [BP, IP, O, IL, O]),
            ([21, 22, 23, 24], [O, BO, BL, IL]),
            ([31, 32, 33], [BL, IL, IL])]
    L = 8
    ids, lab, n = np.zeros((3, L), np.int32), np.zeros((3, L), np.int32), np.zeros(3, np.int32)
    for r, (t, y) in enumerate(rows):
        if bert:
            t, y = [101] + t + [102], [CLS] + y + [SEP]
        ids[r, :len(t)], lab[r, :len(y)], n[r] = t, y, len(t)
    return ids, lab, n


@pytest.mark.parametrize("bert", [True, False])
def test_pool_from_records(tmp_path, bert):
    ids, lab, n = _rows(bert)
    feats = [{'token_ids': ids[r], 'label_ids': lab[r], 'seq_len': int(n[r]), 'mask': (np.arange(8) < n[r]).astype(int),
              'segment_ids': np.zeros(8, int)} for r in range(3)]
    path = str(tmp_path / 'train.nerrec')
    records.write_records(path, feats, 8)
    pool = augment.Pool.from_records(path, MSRA_IDX2TAG)
    assert pool.types == ['LOC', 'ORG', 'PER']
    assert pool.type_tag.tolist() == [[BL, IL], [BO, IO], [BP, IP]]
    assert pool.tag_class[[PAD, O, BL, IL, BO, IO, BP, IP, CLS, SEP]].tolist() == [0, 1, 2, 3, 4, 5, 6, 7, 0, 0]
    # mentions: LOC [23 24], [31 32 33]; ORG [22]; PER [11 12] -- the stray I-LOC (14) is no mention
    assert pool.mention_type_off.tolist() == [0, 2, 3, 4]
    men = [pool.mention_tokens[a:b].tolist() for a, b in zip(pool.mention_tok_off[:-1], pool.mention_tok_off[1:])]
    assert men == [[23, 24], [31, 32, 33], [22], [11, 12]]
    tok = {y: pool.tag_tokens[pool.tag_tok_off[y]:pool.tag_tok_off[y + 1]].tolist() for y in range(10)}
    assert tok[O] == [13, 15, 21] and tok[IL] == [14, 24, 32, 33] and tok[BP] == [11] and tok[IP] == [12]
    assert tok[PAD] == tok[CLS] == tok[SEP] == []
    assert pool.pad_id == 0 and pool.pad_tag == PAD


def test_parse_and_settings():
    assert augment.parse_augment('mr=0.3, lwtr=0.3,sis=0.3,mlm=0.15') == {'mr': .3, 'lwtr': .3, 'sis': .3, 'mlm': .15}
    assert augment.parse_augment('') == {}
    for bad in ('syn=0.3', 'mr=1.5', 'mr=-0.1', 'mr', 'mr=x', 'mr=0.1,mr=0.2', 'mr=nan'):
        with pytest.raises(ValueError):
            augment.parse_augment(bad)
    assert augment.settings({}) is None and augment.settings({'augment': {}}) is None
    s = augment.settings({'augment': {'mr': 0.3}, 'pretrain_dir': 'P'})
    assert s['rows'] == 0.5 and s['temperature'] == 1.0 and s['mlm_dir'] == 'P' and s['probs'] == {'mr': 0.3}
    for bad in ({'augment': {'x': 0.1}}, {'augment': {'mr': 2}}, {'augment': {'mr': 0.1}, 'augment_rows': 1.1},
                {'augment': {'mr': 0.1}, 'augment_mlm_temperature': 0}, {'augment': [0.1]}):
        with pytest.raises(ValueError):
            augment.settings(bad)


def test_step_seed_follows_pretrain():
    assert augment.step_seed(1234, 7) == (1234 * 1000003 + 7) & 0xFFFFFFFFFFFFFFFF
    assert augment.step_seed(-1, 0) < 2 ** 64


def _params(**kw):
    p = {'label_size': 10, 'idx2tag': dict(MSRA_IDX2TAG), 'augment': {'mr': 0.3}}
    p.update(kw)
    return p


@pytest.mark.parametrize("name", ["bilstm_crf_softlexicon", "bilstm_crf_bichar", "bilstm_crf_softword",
                                  "bilstm_crf_ex_softword", "lattice_lstm_crf", "bert_bilstm_crf_softlexicon",
                                  "bert_bilstm_crf_mtl", "bert_bilstm_crf_adv"])
def test_refused_plugins(name):
    with pytest.raises(ValueError, match="cannot augment"):
        engine.Estimator(name, _params(), device='cpu')


def test_refused_teacher_and_label_mask(tmp_path):
    teacher = engine.Estimator('bilstm_crf_softword', {'label_size': 10, 'idx2tag': dict(MSRA_IDX2TAG)}, device='cpu')
    with pytest.raises(ValueError, match="teacher"):
        engine.Estimator('bilstm_crf', _params(), device='cpu', teacher=teacher)
    feats = [{'token_ids': np.ones(4, int), 'label_ids': np.ones(4, int), 'seq_len': 4, 'mask': np.ones(4, int),
              'segment_ids': np.zeros(4, int), 'label_mask': np.full(4, 2)}]
    path = str(tmp_path / 'train.nerrec')
    records.write_records(path, feats, 4)
    with pytest.raises(ValueError, match="label_mask"):
        augment.build(_params(), MSRA_IDX2TAG, path, 'cpu', 'bilstm_crf')
    aug = augment.Augmenter(augment.settings(_params()), augment.Pool.from_arrays(np.ones((1, 4)), np.ones((1, 4)), [4],
                                                                                 MSRA_IDX2TAG), 'cpu')
    with pytest.raises(ValueError, match="label_mask"):
        aug.launch({'label_mask': object()}, 0)


def _bert_dir(path, vocab, head=True):
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, 'vocab.txt'), 'w') as f:
        f.write('\n'.join(vocab) + '\n')
    with open(os.path.join(path, 'bert_config.json'), 'w') as f:
        json.dump({'vocab_size': len(vocab), 'hidden_size': 64, 'num_hidden_layers': 1, 'num_attention_heads': 2,
                   'intermediate_size': 128}, f)
    from chinesener_b200 import mlm, tf_checkpoint
    names = ['bert/embeddings/word_embeddings'] + (mlm.head_names() if head else [])
    tf_checkpoint.save_tf_checkpoint(os.path.join(path, 'bert_model.ckpt'),
                                     {n: np.zeros((2,), np.float32) for n in names})
    return str(path)


VOCAB = ['[PAD]', '[unused1]', '[UNK]', '[CLS]', '[SEP]', '[MASK]', '的', '中', '##国', '人']


def test_refused_mlm(tmp_path):
    tagger = _bert_dir(tmp_path / 'tagger', VOCAB)
    p = _params(augment={'mlm': 0.2}, pretrain_dir=tagger)
    engine.Estimator('bert_crf', p, device='cpu')                       # the tagger's own BERT with its head: accepted
    with pytest.raises(ValueError, match="BERT-tokenized"):
        engine.Estimator('bilstm_crf', p, device='cpu')
    other = _bert_dir(tmp_path / 'other', VOCAB[:-1] + ['们'])
    with pytest.raises(ValueError, match="vocab.txt"):
        engine.Estimator('bert_crf', dict(p, augment_mlm_dir=other), device='cpu')
    headless = _bert_dir(tmp_path / 'headless', VOCAB, head=False)
    with pytest.raises(ValueError, match="masked-LM head"):
        engine.Estimator('bert_crf', dict(p, augment_mlm_dir=headless), device='cpu')
    with pytest.raises(ValueError, match="augment_mlm_dir"):
        engine.Estimator('bert_crf', _params(augment={'mlm': 0.2}, pretrain_dir=''), device='cpu')
    engine.Estimator('bert_crf', _params(augment={'mlm': 0.0}), device='cpu')     # mlm off: nothing to check
    assert augment.eligible_ids({t: i for i, t in enumerate(VOCAB)}).tolist() == [0, 0, 0, 0, 0, 0, 1, 1, 0, 1]


def test_main_parses_augment():
    from chinesener_b200 import main
    args = main.build_parser().parse_args(['--model_name', 'bilstm_crf', '--augment', 'mr=0.3,sis=0.2',
                                           '--augment_rows', '0.7', '--seed', '9'])
    p = {}
    main._augment_params(p, args)
    assert p == {'augment': {'mr': 0.3, 'sis': 0.2}, 'augment_seed': 9, 'augment_rows': 0.7}
    p = {}
    main._augment_params(p, main.build_parser().parse_args(['--model_name', 'bilstm_crf']))
    assert p == {}
    with pytest.raises(ValueError):
        main._augment_params({}, main.build_parser().parse_args(['--model_name', 'x', '--augment', 'syn=0.1']))


# ------------------------------------------------------------------ invariants of the oracle's rules on random rows
def random_batch(B, L, seed, bert=True, K_types=3):
    """Random BIO rows (mentions, stray I-X, O runs), some full-length, some empty, some without entities."""
    rng = np.random.default_rng(seed)
    ids, lab = np.zeros((B, L), np.int32), np.zeros((B, L), np.int32)
    n = np.zeros(B, np.int32)
    for b in range(B):
        want = [L, 0, 1, 2][b] if b < 4 else int(rng.integers(0, L + 1))
        core = want - 2 if bert else want
        toks, tags = [], []
        while len(tags) < core:
            r = rng.random()
            if r < 0.25 and b % 7 != 5:
                x = int(rng.integers(0, K_types))
                ln = int(rng.integers(1, 5))
                tags += [2 + 2 * x] + [3 + 2 * x] * (ln - 1)
            elif r < 0.3 and b % 7 != 5:
                tags.append(3 + 2 * int(rng.integers(0, K_types)))
            else:
                tags += [O] * int(rng.integers(1, 6))
        tags = tags[:max(core, 0)]
        toks = rng.integers(106, 5000, len(tags)).tolist()
        if bert and want >= 2:
            toks, tags = [101] + toks + [102], [CLS] + tags + [SEP]
        elif bert:
            toks, tags = [101][:want], [CLS][:want]
        n[b] = len(toks)
        ids[b, :n[b]], lab[b, :n[b]] = toks, tags
    mask = (np.arange(L)[None] < n[:, None]).astype(np.int32)
    return ids, lab, n, mask, np.zeros((B, L), np.int32)


def _pool(seed=3, bert=True):
    ids, lab, n, _, _ = random_batch(64, 40, seed, bert)
    return augment.Pool.from_arrays(ids, lab, n, MSRA_IDX2TAG)


def _mentions(tags, pool):
    return [(tags[s], ln) for s, ln in ao.segments(tags, pool.tag_class, pool.type_tag) if 2 <= pool.tag_class[tags[s]] and
            pool.tag_class[tags[s]] % 2 == 0]


@pytest.mark.parametrize("bert", [True, False])
def test_oracle_invariants(bert):
    pool = _pool(bert=bert)
    L = 24
    ids, lab, n, mask, seg = random_batch(48, L, 11, bert)
    seed = 0xABCDEF0123
    specials = lambda y: [(t, v) for t, v in enumerate(y) if pool.tag_class[v] == 0]
    for probs in [(1, 1, 0, 0, 0), (1, 0, 0, 1, 0), (1, 0.5, 0.5, 0.5, 0.5)]:
        out = ao.augment_rows(ids, lab, n, mask, seg, pool, probs, seed, mask_id=103, mlm=True)
        for b in range(len(n)):
            m0, m1 = int(n[b]), int(out['seq_len'][b])
            y0, y1 = lab[b, :m0].tolist(), out['label_ids'][b, :m1].tolist()
            assert m1 <= L                                                            # the length cap holds
            assert out['mask'][b].tolist() == [1] * m1 + [0] * (L - m1)
            s0, s1 = specials(y0), specials(y1)                                      # specials untouched, [SEP] moves
            assert [v for _, v in s0] == [v for _, v in s1]
            if bert and m0 >= 2:
                assert y1[0] == CLS and y1[-1] == SEP and out['token_ids'][b, 0] == 101 and out['token_ids'][b, m1 - 1] == 102
            # MR keeps the mentions per type and the order of the non-mention tags
            assert Counter(t for t, _ in _mentions(y0, pool)) == Counter(t for t, _ in _mentions(y1, pool))
            non = lambda y: [y[s:s + ln] for s, ln in ao.segments(y, pool.tag_class, pool.type_tag)
                             if not (pool.tag_class[y[s]] >= 2 and pool.tag_class[y[s]] % 2 == 0)]
            assert non(y0) == non(y1)
            if probs[1] == 0:
                assert y0 == y1
            pos = [p for p in out['mlm_positions'][b] if p >= 0]
            assert len(pos) <= ao.BUDGET and all(y1[p - b * L] == O for p in pos)
            assert all(out['mlm_ids'][b, p - b * L] == 103 for p in pos)
        if probs == (1, 0, 0, 1, 0):                                                   # SiS keeps each segment's multiset
            for b in range(len(n)):
                m = int(n[b])
                for s, ln in ao.segments(lab[b, :m].tolist(), pool.tag_class, pool.type_tag):
                    assert sorted(ids[b, s:s + ln]) == sorted(out['token_ids'][b, s:s + ln])
            assert (out['token_ids'] != ids).any()


def test_oracle_noop_and_skip_rule():
    pool = _pool()
    ids, lab, n, mask, seg = random_batch(32, 24, 5)
    for probs in [(0, 1, 1, 1, 1), (1, 0, 0, 0, 0)]:
        out = ao.augment_rows(ids, lab, n, mask, seg, pool, probs, 99)
        for k, v in (('token_ids', ids), ('label_ids', lab), ('seq_len', n), ('mask', mask), ('segment_ids', seg)):
            assert (out[k] == v).all(), (probs, k)
    # a full-length row whose mentions are all chosen: any longer replacement is skipped, the row never exceeds L
    out = ao.augment_rows(ids[:1], lab[:1], n[:1], mask[:1], seg[:1], pool, (1, 1, 0, 0, 0), 7)
    assert n[0] == 24 and out['seq_len'][0] <= 24
