"""GPU: the CRF plugins on a 108-tag set (52 entity types in BIO plus the specials), through the wide CRF kernels and the
split-bf16 logits projection: PREDICT / EVAL against the oracle models, TRAIN lowers the loss, GPU span extraction past
32 types equals extract_entity, and what stops at 32 tags is refused before a launch."""
import json

import numpy as np
import pytest
import torch

from chinesener_b200 import engine, ops, synthetic, variables
from chinesener_b200.tools.infer_utils import extract_entity, extract_entity_device
from oracle import crf, models as omodels

pytestmark = pytest.mark.gpu

K = 108
TYPES = ['T%02d' % i for i in range(52)]
IDX2TAG = dict(enumerate(['[PAD]', 'O'] + [p + '-' + t for t in TYPES for p in ('B', 'I')] + ['[CLS]', '[SEP]']))
SMALL_BERT = {'vocab_size': 3000, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
              'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02}


def _params(L):
    p = synthetic.data_params(L, label_size=K)
    p['idx2tag'] = dict(IDX2TAG)
    p['tag2idx'] = {v: k for k, v in IDX2TAG.items()}
    return p


def _batch(B, L, vocab, seed):
    feats = synthetic.msra_batch(B, L, vocab=vocab, seed=seed)
    rng = np.random.default_rng(seed)
    lab = rng.integers(1, K - 2, size=(B, L)).astype(np.int32)
    lens = feats['seq_len'].numpy()
    for b in range(B):
        lab[b, lens[b]:] = 0
        lab[b, 0], lab[b, lens[b] - 1] = K - 2, K - 1
    feats['label_ids'] = torch.from_numpy(lab)
    return feats


def _bert_est(model_name, tmp_path, L):
    (tmp_path / "bert_config.json").write_text(json.dumps(SMALL_BERT))
    return engine.Estimator(model_name, dict(_params(L), pretrain_dir=str(tmp_path)))


@pytest.mark.parametrize("model_name", ["bert_bilstm_crf", "bert_crf"])
def test_bert_plugins_match_oracle_at_108_tags(model_name, tmp_path):
    B, L = 6, 48
    feats = _batch(B, L, SMALL_BERT['vocab_size'], seed=5)
    est = _bert_est(model_name, tmp_path, L)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(8.0)
    est.store.touch()
    dev = est.to_device(feats)
    loss, pred = est.forward_device(dev)
    pred = pred.cpu().numpy()
    w = est.store.state_dict()
    p = dict(est.params, num_hidden_layers=2, num_attention_heads=12)
    ref = getattr(omodels, model_name)(w, feats, p, dtype=torch.float64, emulate_bf16=True)
    from chinesener_b200.tools import layer
    with variables.use_store(est.store):
        emb = layer.pretrain_bert_embedding(dev['token_ids'], dev['mask'], dev['segment_ids'], est.params['pretrain_dir'],
                                            0.1, False)
        x = layer.bilstm(emb, 'lstm', est.params['rnn_activation'], [128], [1.0], 1, dev['seq_len'], 'float32',
                         False) if model_name == "bert_bilstm_crf" else emb
        logits = layer.dense(x, K, 'logits')
    assert logits.shape == (B, L, K)
    valid = (torch.arange(L)[None, :] < feats['seq_len'][:, None])
    err = (logits.cpu().double() - ref['logits'])[valid].abs().max().item()
    assert err < 4e-3 * max(1.0, ref['logits'][valid].abs().max().item())
    trans = w['crf_layer/transitions'].numpy()
    ref_pred, _ = crf.crf_decode(logits.cpu().numpy(), trans, feats['seq_len'].numpy(), dtype=np.float32)
    np.testing.assert_array_equal(pred, ref_pred)                    # Viterbi on the CUDA logits: bit-exact
    ll_ref = crf.crf_log_likelihood(logits.cpu().numpy(), feats['label_ids'].numpy(), feats['seq_len'].numpy(), trans)
    assert abs(float(loss) - float(np.mean(-ll_ref))) < 1e-3 * max(1.0, abs(float(loss)))
    assert (pred == ref['pred_ids']).mean() > 0.99
    assert est.predict_device(dev).shape == (B, L)                   # the fused executor steps aside above 32 tags


def _bilstm_est(L, V=3000):
    g = torch.Generator().manual_seed(0)
    emb = torch.nn.functional.normalize(torch.randn(V, 50, generator=g), dim=1).numpy()
    return engine.Estimator("bilstm_crf", dict(_params(L), embedding=emb))


def test_bilstm_crf_matches_oracle_and_trains_at_108_tags():
    B, L = 8, 40
    feats = _batch(B, L, 3000, seed=2)
    est = _bilstm_est(L)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(6.0)
    est.store.touch()
    out = est.evaluate(feats)
    ref = omodels.bilstm_crf(est.store.state_dict(), feats, est.params, dtype=torch.float64, emulate_bf16=True)
    assert abs(out['loss'] - ref['loss']) < 2e-3 * max(1.0, abs(ref['loss']))
    assert (out['pred_ids'].numpy() == ref['pred_ids']).mean() > 0.99
    first = float(est.train_step(feats))
    for _ in range(40):
        last = float(est.train_step(feats))
    assert np.isfinite(last) and last < 0.7 * first, (first, last)
    assert est.store.vars['crf_layer/transitions'].shape == (K, K)
    assert est.store.vars['logits/kernel'].shape[1] == K


def test_span_extraction_past_32_types():
    rng = np.random.default_rng(3)
    B, L = 40, 60
    pred = rng.integers(0, K, size=(B, L)).astype(np.int32)
    pred[:, 0] = 0
    toks = [[chr(0x4e00 + (b * L + t) % 500) for t in range(L)] for b in range(B)]
    got = extract_entity_device(toks, torch.from_numpy(pred).cuda(), IDX2TAG)
    for b in range(B):
        assert dict(got[b]) == dict(extract_entity(toks[b], pred[b].tolist(), IDX2TAG)), b
    assert any(t >= 'T32' for ent in got for t in ent)             # types past index 31 come back with their names
    table, _ = ops.tag_classes(IDX2TAG)
    assert table.dtype == torch.int16


class _NoTensor(dict):
    def __getitem__(self, k):
        raise AssertionError("read {!r} before refusing".format(k))

    def get(self, k, default=None):
        if k == 'label_mask':
            return True
        raise AssertionError("read {!r} before refusing".format(k))


def test_refusals_above_32_tags(tmp_path):
    L = 16
    before = torch.cuda.memory_allocated()
    est = _bilstm_est(L)
    with pytest.raises(ValueError, match="32 tags"):
        est.train_step(_NoTensor())
    est.params['crf_nbest'] = 2
    with pytest.raises(ValueError, match="at most 32 tags"):
        est.crf_nbest()
    with pytest.raises(ValueError, match="at most 32 tags"):
        engine.Estimator("bilstm_crf", dict(_params(L), embedding=np.zeros((10, 4), np.float32)), teacher=_bilstm_est(L))
    for plugin in ("bert_ce", "bert_dice"):
        with pytest.raises(ValueError, match="at most 32 tags"):
            _bert_est(plugin, tmp_path, L)
    assert torch.cuda.memory_allocated() == before                   # nothing was placed on the device
