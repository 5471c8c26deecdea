"""GPU: ner_augment_rows bit for bit against the oracle, ner_vocab_sample against a float64 Gumbel-max and softmax(z / T),
the no-op and off cases, determinism, the pipelined path, and training with every operation on."""
import json

import numpy as np
import pytest
import torch

import _augment_oracle as ao
from chinesener_b200 import augment, bert, engine, main, mlm, ops, synthetic, variables
from chinesener_b200.synthetic import MSRA_IDX2TAG
from test_augment_host import random_batch

pytestmark = pytest.mark.gpu

OPS_ALONE = {'mr': (1, .5, 0, 0, 0), 'lwtr': (1, 0, .5, 0, 0), 'sis': (1, 0, 0, .5, 0), 'mlm': (1, 0, 0, 0, .3),
             'all': (.7, .4, .3, .5, .3), 'every': (1, 1, 1, 1, 1)}


def _pool(bert_rows, seed=3):
    ids, lab, n, _, _ = random_batch(96, 40, seed, bert_rows)
    return augment.Pool.from_arrays(ids, lab, n, MSRA_IDX2TAG)


def _run(pool, batch, probs, seed, mlm_on=True):
    d = [torch.from_numpy(a).cuda() for a in batch]
    out = ops.augment_rows(*d, pool.tables('cuda'), probs, seed, pool.pad_id, pool.pad_tag, 103, want_mlm=mlm_on)
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("op", list(OPS_ALONE))
@pytest.mark.parametrize("bert_rows", [True, False])
@pytest.mark.parametrize("L", [127, 128, 512])
def test_rows_match_the_oracle(op, bert_rows, L):
    pool = _pool(bert_rows)
    batch = random_batch(67, L, 17 + L, bert_rows)
    seed = 0x0123_4567_89AB_CDEF
    got = _run(pool, batch, OPS_ALONE[op], seed)
    ref = ao.augment_rows(*batch, pool, OPS_ALONE[op], seed, mask_id=103, mlm=True)
    for k in ref:
        assert (got[k] == ref[k]).all(), k
    if op != 'mlm':
        assert (got['token_ids'] != batch[0]).any()
    if op in ('mr', 'every'):
        assert (got['seq_len'] != batch[2]).any()


def test_long_rows_and_a_short_pool():
    """L = 4095 document rows, and a full-length row whose replacements must all be skipped."""
    pool = _pool(True)
    batch = random_batch(5, 4095, 1, True)
    got = _run(pool, batch, OPS_ALONE['every'], 77)
    ref = ao.augment_rows(*batch, pool, OPS_ALONE['every'], 77, mask_id=103, mlm=True)
    for k in ref:
        assert (got[k] == ref[k]).all(), k
    assert got['seq_len'][0] <= 4095


@pytest.mark.parametrize("probs", [(0, 1, 1, 1, 1), (1, 0, 0, 0, 0)])
def test_noop_is_byte_identical(probs):
    pool = _pool(True)
    batch = random_batch(40, 128, 4, True)
    got = _run(pool, batch, probs, 5)
    for k, v in zip(('token_ids', 'label_ids', 'seq_len', 'mask', 'segment_ids'), batch):
        assert (got[k] == v).all(), k


def test_determinism():
    pool = _pool(True)
    batch = random_batch(40, 128, 4, True)
    s1, s2 = augment.step_seed(1234, 10), augment.step_seed(1234, 11)
    a, b, c = _run(pool, batch, OPS_ALONE['all'], s1), _run(pool, batch, OPS_ALONE['all'], s1), _run(pool, batch,
                                                                                                  OPS_ALONE['all'], s2)
    assert all((a[k] == b[k]).all() for k in a)
    assert (a['token_ids'] != c['token_ids']).any()


def test_sampler_matches_float64_gumbel_max():
    rng = np.random.default_rng(0)
    M, V, ld = 300, 2003, 2004
    logits = (rng.standard_normal((M, ld)) * 3).astype(np.float32)
    elig = (rng.random(V) < 0.8).astype(np.uint8)
    B, L = 20, 64
    toks = rng.integers(0, V, (B, L)).astype(np.int32)
    pos = rng.choice(B * L, M, replace=False).astype(np.int32)
    pos[::7] = -1
    seed, T = 0xFEED_0000_1234, 0.8
    out = torch.from_numpy(toks.copy()).cuda()
    ops.vocab_sample(torch.from_numpy(logits).cuda(), V, torch.from_numpy(elig).cuda(), torch.from_numpy(pos).cuda(), out,
                     T, seed)
    got = out.cpu().numpy().reshape(-1)
    flat = toks.reshape(-1)
    untouched = np.ones(B * L, bool)
    checked = 0
    for r in range(M):
        p = int(pos[r])
        if p < 0:
            continue
        untouched[p] = False
        s = ao.gumbel_scores(logits[r], V, elig, int(flat[p]), p, T, seed)
        top2 = np.sort(s)[-2:]
        j = int(got[p])
        assert elig[j] and j != flat[p]
        if top2[1] - top2[0] > 1e-4:
            assert j == int(np.argmax(s)), r
            checked += 1
    assert checked > M * 0.8
    assert (got[untouched] == flat[untouched]).all()


def test_sampler_follows_the_tempered_softmax():
    from scipy.stats import chisquare
    z = np.array([1.0, 0.2, -0.5, 2.0, 0.0, -1.0, 0.7, 1.5], np.float32)
    elig = np.array([1, 1, 0, 1, 1, 1, 1, 1], np.uint8)
    V, T, M = 8, 0.7, 20000
    for seed in (1, 2, 3):
        toks = torch.full((M,), 6, dtype=torch.int32, device='cuda')          # original id 6: excluded
        logits = torch.from_numpy(np.tile(z, (M, 1))).cuda()
        ops.vocab_sample(logits, V, torch.from_numpy(elig).cuda(), torch.arange(M, dtype=torch.int32, device='cuda'),
                         toks, T, seed)
        counts = np.bincount(toks.cpu().numpy(), minlength=V)
        ok = (elig == 1) & (np.arange(V) != 6)
        assert counts[~ok].sum() == 0
        p = np.exp(z[ok].astype(np.float64) / T)
        assert chisquare(counts[ok], p / p.sum() * counts[ok].sum()).pvalue > 1e-3, seed


# ------------------------------------------------------------------ through the Estimator
def _emb(V=2000, E=32):
    return np.random.default_rng(0).standard_normal((V, E)).astype(np.float32) * 0.1


def _bilstm(**kw):
    p = dict(synthetic.data_params(32), embedding=_emb(), embedding_dropout=0.0, keep_prob_list=[1.0])
    p.update(kw)
    store = variables.VariableStore('cuda', seed=7)
    return engine.Estimator('bilstm_crf', p, store=store)


def _host_pool():
    b = synthetic.msra_batch(256, 32, vocab=2000, seed=99)
    return augment.Pool.from_arrays(b['token_ids'].numpy(), b['label_ids'].numpy(), b['seq_len'].numpy(), MSRA_IDX2TAG)


def _augmenter(probs, pool=None, mlm=None, rows=1.0):
    s = augment.settings({'augment': probs, 'augment_rows': rows, 'augment_seed': 5})
    return augment.Augmenter(s, pool or _host_pool(), 'cuda', mlm)


def test_noop_train_step_is_bit_identical():
    batch = synthetic.msra_batch(32, 32, vocab=2000, seed=1)
    est = _bilstm()
    ref = float(est.train_step(batch))
    for probs, rows in (({'mr': 0, 'lwtr': 0, 'sis': 0}, 1.0), ({'mr': 1, 'lwtr': 1, 'sis': 1}, 0.0)):
        est2 = _bilstm()
        dev = _augmenter(probs, rows=rows).augment(est2.to_device(batch), 0)
        assert float(est2.train_step(dev)) == ref


def test_pipeline_equals_direct_path():
    aug = _augmenter({'mr': .3, 'lwtr': .3, 'sis': .3})
    est = _bilstm()
    batches = [synthetic.msra_batch(32, 32, vocab=2000, seed=s) for s in range(4)]
    piped = list(aug.pipeline(iter(batches), 40, est.to_device))
    for i, (h, p) in enumerate(zip(batches, piped)):
        d = aug.augment(est.to_device(h), 40 + i)
        for k in augment.AUGMENTED:
            assert torch.equal(p[k], d[k]), (i, k)
        assert (p['mask'].row_lengths == d['mask'].row_lengths).all()
        assert p['mask'].total_tokens == d['mask'].total_tokens and p['mask'].nonempty_rows == d['mask'].nonempty_rows
        assert (d['mask'].row_lengths == d['seq_len'].cpu().numpy()).all()


class _Pipe:
    """A two-batch train split in memory for main.train_and_evaluate."""

    def __init__(self, path):
        self.path = path

    def file_path(self, name):
        return self.path

    def build_input_fn(self, name, is_predict=0, with_strings=None):
        return lambda: iter([synthetic.msra_batch(32, 32, vocab=2000, seed=s) for s in range(2)])


def _records(tmp_path):
    from chinesener_b200.data import records
    b = synthetic.msra_batch(64, 32, vocab=2000, seed=3)
    feats = [{k: b[k][r].numpy() if b[k].dim() > 1 else int(b[k][r]) for k in ('token_ids', 'label_ids', 'mask',
                                                                                'segment_ids', 'seq_len')}
             for r in range(64)]
    path = str(tmp_path / 'train.nerrec')
    records.write_records(path, feats, 32)
    return path


@pytest.mark.parametrize("on", [False, True])
def test_train_and_evaluate_runs_augmentation_only_when_set(tmp_path, monkeypatch, on):
    calls = []
    real = ops.augment_rows

    def spy(*a, **k):
        if not on:
            raise AssertionError("augmentation ran with augment unset")
        calls.append(1)
        return real(*a, **k)
    monkeypatch.setattr(ops, 'augment_rows', spy)
    monkeypatch.setattr(ops, 'vocab_sample', lambda *a, **k: (_ for _ in ()).throw(AssertionError("vocab_sample ran")))
    est = _bilstm(**({'augment': {'mr': .3, 'lwtr': .3, 'sis': .3}} if on else {}))
    hist = main.train_and_evaluate(est, _Pipe(_records(tmp_path)), str(tmp_path / 'ck'), log=lambda *a: None)
    assert hist['final_step'] == 2
    assert len(calls) == (2 if on else 0)


def _losses(est, aug, steps, B=32, L=32, vocab=2000):
    batches = [synthetic.msra_batch(B, L, vocab=vocab, seed=s) for s in range(4)]
    out = []
    for i, dev in enumerate(aug.pipeline((batches[i % 4] for i in range(steps)), 0, est.to_device)):
        out.append(float(est.train_step(dev)))
    return np.array(out)


def test_bilstm_crf_trains_with_augmentation():
    est = _bilstm(lr=0.01)
    loss = _losses(est, _augmenter({'mr': .3, 'lwtr': .3, 'sis': .3}, rows=0.5), 100)
    assert np.isfinite(loss).all() and loss[-10:].mean() < loss[:10].mean()


def test_bilstm_crf_distils_with_augmentation():
    p = dict(synthetic.data_params(32), embedding=_emb(), embedding_dropout=0.0, keep_prob_list=[1.0])
    teacher = engine.Estimator('bilstm_crf', p)
    teacher.evaluate(synthetic.msra_batch(32, 32, vocab=2000, seed=0))
    student = engine.Estimator('bilstm_crf', dict(p, augment={'mr': .3, 'lwtr': .3, 'sis': .3}), teacher=teacher)
    loss = _losses(student, _augmenter({'mr': .3, 'lwtr': .3, 'sis': .3}), 30)
    assert np.isfinite(loss).all()


TINY = {'vocab_size': 1000, 'hidden_size': 128, 'num_hidden_layers': 2, 'num_attention_heads': 2, 'intermediate_size': 512,
        'max_position_embeddings': 64, 'type_vocab_size': 2, 'initializer_range': 0.02, 'hidden_dropout_prob': 0.0,
        'attention_probs_dropout_prob': 0.0}


def _tiny_bert_with_head(tmp_path):
    """A 1000-token vocab.txt, the tiny config and a checkpoint with the masked-LM head."""
    d = tmp_path / 'bert'
    d.mkdir()
    (d / 'bert_config.json').write_text(json.dumps(TINY))
    vocab = ['[PAD]'] + ['[unused%d]' % i for i in range(1, 100)] + ['[UNK]', '[CLS]', '[SEP]', '[MASK]', '##x']
    vocab += [chr(0x4E00 + i) for i in range(1000 - len(vocab))]
    (d / 'vocab.txt').write_text('\n'.join(vocab) + '\n')
    cfg = bert.load_bert_config(str(d))
    store = variables.VariableStore('cuda', seed=3)
    with pytest.warns(UserWarning):
        bert.create_bert_variables(cfg, store)
    mlm.create_head_variables(cfg, store)
    mlm.export_pretrained(store, str(d), str(d))
    return str(d)


@pytest.mark.parametrize("model", ["bert_crf", "bert_global_pointer"])
def test_bert_plugins_train_with_every_operation(tmp_path, model):
    d = _tiny_bert_with_head(tmp_path)
    probs = {'mr': .3, 'lwtr': .3, 'sis': .3, 'mlm': .15}
    params = dict(synthetic.data_params(32), pretrain_dir=d, augment=probs, augment_seed=5, lr=5e-4, num_train_steps=100)
    est = engine.Estimator(model, params, store=variables.VariableStore('cuda', seed=7))
    pool = augment.Pool.from_arrays(*(synthetic.msra_batch(256, 32, vocab=1000, seed=99)[k].numpy()
                                      for k in ('token_ids', 'label_ids', 'seq_len')), MSRA_IDX2TAG)
    aug = augment.Augmenter(augment.settings(params), pool, 'cuda',
                            augment.FrozenMLM(d, augment.mlm_vocab(d, d, 'bert'), 1.0, 'cuda'))
    loss = _losses(est, aug, 100, vocab=1000)
    assert np.isfinite(loss).all() and loss[-10:].mean() < loss[:10].mean()


def test_mlm_replacement_draws_eligible_ids_at_the_masked_positions(tmp_path):
    d = _tiny_bert_with_head(tmp_path)
    vocab = augment.mlm_vocab(d, d, 'bert')
    frozen = augment.FrozenMLM(d, vocab, 1.0, 'cuda')
    aug = _augmenter({'mlm': 0.5}, pool=augment.Pool.from_arrays(
        *(synthetic.msra_batch(64, 32, vocab=1000, seed=9)[k].numpy() for k in ('token_ids', 'label_ids', 'seq_len')),
        MSRA_IDX2TAG), mlm=frozen)
    host = synthetic.msra_batch(32, 32, vocab=1000, seed=4)
    dev = {k: v.cuda() for k, v in host.items()}
    out = aug.augment(dev, 3)
    seed = augment.step_seed(5, 3)
    ref = ao.augment_rows(*(host[k].numpy() for k in ('token_ids', 'label_ids', 'seq_len', 'mask', 'segment_ids')),
                          aug.pool, aug.probs, seed, mask_id=vocab['[MASK]'], mlm=True)
    got = out['token_ids'].cpu().numpy()
    pos = ref['mlm_positions'][ref['mlm_positions'] >= 0]
    assert len(pos) > 20
    elig = augment.eligible_ids(vocab)
    flat_ref, flat_got = ref['token_ids'].reshape(-1), got.reshape(-1)
    assert all(elig[flat_got[p]] and flat_got[p] != flat_ref[p] for p in pos)
    other = np.ones(flat_ref.shape, bool)
    other[pos] = False
    assert (flat_got[other] == flat_ref[other]).all()
    assert (out['label_ids'].cpu().numpy() == ref['label_ids']).all()
