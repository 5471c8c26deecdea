# -*-coding:utf-8 -*-
"""GPU: the bert_mrc plugin (MRC-style NER, one BERT query per entity type) and its kernels ner_mrc_pairs / ner_mrc_merge.

  * ner_mrc_pairs: every output bit-exact vs the numpy restatement (tests/_mrc_oracle.py) for T in {1, 3, 32}, ragged and
    zero-length queries, seq_len in {0, 1, 2, L}; nothing written past the outputs;
  * ner_mrc_merge: bit-exact vs the float32 restatement away from near-ties, the tie rule, the fixed positions, and on
    overlap-free inputs the entities of the merged tags are the union of the per-type entities;
  * plugin PREDICT / EVAL vs a float64 restatement (pairs -> BertModel -> dense -> alignment -> CE -> merge, bf16
    emulated), TRAIN gradients vs float64 autograd (packed and padded encoder), a short AdamW run, the driver pickle,
    InferHelper, and no device-to-host synchronisation in PREDICT.
"""
import ctypes
import json
import os
import pickle

import numpy as np
import pytest
import torch

from _mrc_oracle import mrc_merge as oracle_merge
from _mrc_oracle import mrc_pairs as oracle_pairs
from chinesener_b200 import _lib, autodiff, engine, evaluation, ops, synthetic, variables
from chinesener_b200.data import mrc
from chinesener_b200.tools.infer_utils import extract_entity
from oracle import nn as onn

pytestmark = pytest.mark.gpu

SMALL_BERT = {'vocab_size': 3000, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
              'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02}
MSRA_IDX2TAG = synthetic.MSRA_IDX2TAG
QUERY_LENS = {'ORG': 22, 'PER': 10, 'LOC': 20}          # the default queries' token counts


def _query_ids(seed=7, vocab=3000):
    rng = np.random.default_rng(seed)
    return {n: rng.integers(106, vocab, size=k).tolist() for n, k in QUERY_LENS.items()}


# --------------------------------------------------------------------------- ner_mrc_pairs
def _pairs_case(B, L, T, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, L + 1, size=B).astype(np.int32)
    lens[:4] = [0, 1, 2, L]
    token_ids = np.zeros((B, L), np.int32)
    label_ids = np.zeros((B, L), np.int32)
    for b in range(B):
        n = lens[b]
        token_ids[b, :n] = rng.integers(106, 21128, size=n)
        label_ids[b, :n] = rng.integers(0, 2 * T + 2, size=n)
    qlen = rng.integers(0, 9, size=T).astype(np.int32)
    qlen[0] = 0 if T > 1 else 3
    Qmax = int(qlen.max()) + 2                       # a wider table than the longest query
    qids = rng.integers(106, 21128, size=(T, Qmax)).astype(np.int32)
    type_tag = np.array([[2 + 2 * t, 3 + 2 * t] for t in range(T)], np.int32)
    return token_ids, lens, label_ids, qids, qlen, type_tag


@pytest.mark.parametrize("T", [1, 3, 32])
def test_mrc_pairs_bit_exact_with_guards(T):
    B, L = 9, 24
    token_ids, lens, label_ids, qids, qlen, type_tag = _pairs_case(B, L, T, seed=T)
    Qmax = qids.shape[1]
    L2 = Qmax + 1 + L + 3                            # wider than needed: the extra columns are zero too
    ref = oracle_pairs(token_ids, lens, qids, qlen, type_tag, L2, 102, label_ids)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    tok, sl, lab, q, ql, tt = (dev(a) for a in (token_ids, lens, label_ids, qids, qlen, type_tag))
    guard, sentinel = 37, -7
    sizes = dict(ids=B * T * L2, segment_ids=B * T * L2, mask=B * T * L2, seq_len=B * T, labels=B * T * L, align=B * T * L)
    bufs = {k: torch.full((n + guard,), sentinel, dtype=torch.int32, device='cuda') for k, n in sizes.items()}
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    rc = _lib.lib().ner_mrc_pairs(p(tok), p(sl), p(lab), p(q), p(ql), p(tt), B, L, T, Qmax, L2, 102, p(bufs['ids']),
                                  p(bufs['segment_ids']), p(bufs['mask']), p(bufs['seq_len']), p(bufs['labels']),
                                  p(bufs['align']), None)
    assert rc == 0
    torch.cuda.synchronize()
    for k, n in sizes.items():
        got = bufs[k].cpu().numpy()
        np.testing.assert_array_equal(got[:n], ref[k].reshape(-1), err_msg=k)
        assert (got[n:] == sentinel).all(), k
    # the ops wrapper; without label_ids no labels
    out = ops.mrc_pairs(tok, sl, q, ql, tt, L2, 102, label_ids=lab)
    for k in sizes:
        np.testing.assert_array_equal(out[k].cpu().numpy().reshape(-1), ref[k].reshape(-1), err_msg=k)
    assert ops.mrc_pairs(tok, sl, q, ql, tt, L2, 102)['labels'] is None
    empty = ops.mrc_pairs(tok[:0], sl[:0], q, ql, tt, L2, 102)
    assert empty['ids'].shape == (0, L2) and empty['align'].numel() == 0


# --------------------------------------------------------------------------- ner_mrc_merge
def _merge_case(B, L, T, seed):
    rng = np.random.default_rng(seed)
    z = (rng.normal(size=(B, T, L, 3)) * 3).astype(np.float32)
    lens = rng.integers(0, L + 1, size=B).astype(np.int32)
    lens[:4] = [0, 1, 2, L]
    type_tag = [[2 + 2 * t, 3 + 2 * t] for t in range(T)]
    return z, lens, type_tag


def _separate(z, lens, type_tag):
    """Positions whose decision is within 1e-4 of flipping get an unambiguous O row for every type."""
    B, T, L, _ = z.shape
    _, margin = oracle_merge(z.reshape(B * T, L, 3), lens, type_tag, 1, 8, 9)
    near = margin <= 1e-4
    z[np.broadcast_to(near[:, None, :], (B, T, L))] = np.array([2.0, 0.0, 0.0], np.float32)
    return z


@pytest.mark.parametrize("B,L,T", [(6, 7, 1), (33, 40, 3), (5, 128, 32)])
def test_mrc_merge_bit_exact(B, L, T):
    z, lens, type_tag = _merge_case(B, L, T, seed=B + T)
    z = _separate(z, lens, type_tag)
    ref, _ = oracle_merge(z.reshape(B * T, L, 3), lens, type_tag, 1, 8, 9)
    tt = torch.tensor(type_tag, dtype=torch.int32, device='cuda')
    pred = ops.mrc_merge(torch.from_numpy(z.reshape(B * T, L, 3)).cuda(), torch.from_numpy(lens).cuda(), tt, 1, 8, 9)
    got = pred.cpu().numpy()
    np.testing.assert_array_equal(got, ref)
    for b in range(B):
        n = lens[b]
        assert (got[b, n:] == 0).all()
        if n >= 1:
            assert got[b, 0] == 8
        if n >= 2:
            assert got[b, n - 1] == 9


def test_mrc_merge_ties_go_to_the_lower_type():
    B, L, T = 8, 30, 4
    z, lens, type_tag = _merge_case(B, L, T, seed=3)
    z[:] = z[:, :1]                                   # every type sees the same logits: every claim ties
    tt = torch.tensor(type_tag, dtype=torch.int32, device='cuda')
    got = ops.mrc_merge(torch.from_numpy(z.reshape(B * T, L, 3)).cuda(), torch.from_numpy(lens).cuda(), tt, 1, 8, 9).cpu().numpy()
    a = z[:, 0].argmax(-1)
    for b in range(B):
        for s in range(1, lens[b] - 1):
            assert got[b, s] == (1 if a[b, s] == 0 else type_tag[0][a[b, s] - 1])
    np.testing.assert_array_equal(got, oracle_merge(z.reshape(B * T, L, 3), lens, type_tag, 1, 8, 9)[0])


def test_merged_entities_are_the_union_of_the_per_type_entities():
    rng = np.random.default_rng(11)
    idx2tag = dict(MSRA_IDX2TAG)
    types = mrc.entity_types(idx2tag)
    T, B, L = len(types), 16, 48
    lens = rng.integers(2, L + 1, size=B).astype(np.int32)
    z = np.zeros((B, T, L, 3), np.float32)
    z[..., 0] = 4.0                                   # every type says O ...
    per_type = np.zeros((B, T, L), np.int32)          # ... except on its own, non-overlapping spans
    for b in range(B):
        s = 1
        while s < lens[b] - 1:
            k = int(rng.integers(1, 5))
            if rng.random() < 0.4 and s + k <= lens[b] - 1:
                t = int(rng.integers(0, T))
                per_type[b, t, s] = 1
                per_type[b, t, s + 1:s + k] = 2
                s += k + int(rng.integers(0, 2))
            else:
                s += 1
    for c in (1, 2):
        z[..., c] = np.where(per_type == c, 6.0 + rng.random(per_type.shape), 0.0)
    tt = torch.tensor([[bi, ii] for _, bi, ii in types], dtype=torch.int32, device='cuda')
    got = ops.mrc_merge(torch.from_numpy(z.reshape(B * T, L, 3)).cuda(), torch.from_numpy(lens).cuda(), tt, 1, 8, 9).cpu().numpy()
    for b in range(B):
        n = int(lens[b])
        tokens = [chr(0x4e00 + 37 * b + s) for s in range(n)]
        merged = extract_entity(tokens, got[b, :n].tolist(), idx2tag)
        union = {}
        for t, (name, bi, ii) in enumerate(types):
            seq = [8] + [{0: 1, 1: bi, 2: ii}[int(c)] for c in per_type[b, t, 1:n - 1]] + [9]
            for typ, found in extract_entity(tokens, seq, idx2tag).items():
                union.setdefault(typ, set()).update(found)
        assert dict(merged) == union, b
    assert any(per_type.any(axis=(1, 2)))


# --------------------------------------------------------------------------- float64 restatement of the plugin
def masked_token_xent(logits, labels, seq_len):
    B, L, _ = logits.shape
    valid = torch.arange(L)[None, :] < seq_len.long()[:, None]
    ce = torch.logsumexp(logits, -1) - logits.gather(-1, labels.long().clamp(min=0)[..., None])[..., 0]
    n = int(valid.sum())
    return (ce * valid).sum() / n if n > 0 else (ce * 0.0).sum()


def _oracle_pairs(features, table, L2):
    qids = table.query_ids.cpu().numpy()
    qlen = table.query_len.cpu().numpy()
    tt = table.type_tag.cpu().numpy()
    return oracle_pairs(features['token_ids'].numpy(), features['seq_len'].numpy(), qids, qlen, tt, L2, table.sep_id,
                        features['label_ids'].numpy())


def bert_mrc_oracle(w, features, table, num_layers=2, dtype=torch.float64, emulate_bf16=False):
    """pairs -> BertModel -> sentence alignment -> dense 'logits' [B*T, L, 3] -> masked CE over the pairs; pred_ids by the
    merge rule on the float32-rounded logits, with its decision margin."""
    B, L = features['token_ids'].shape
    pr = _oracle_pairs(features, table, table.L2)
    t = lambda a: torch.from_numpy(a)
    seq = onn.bert_encoder(w, t(pr['ids']), t(pr['mask']), t(pr['segment_ids']), num_layers=num_layers, num_heads=12,
                           dtype=dtype, emulate_bf16=emulate_bf16)
    H = seq.shape[-1]
    rows = seq.reshape(-1, H)[t(pr['align']).long()].view(B * table.T, L, H)
    logits = onn.dense(onn._rb(rows, emulate_bf16), w["logits/kernel"].to(dtype), w["logits/bias"].to(dtype))
    loss = masked_token_xent(logits, t(pr['labels']), t(pr['seq_len']))
    pred, margin = oracle_merge(logits.detach().float().numpy(), features['seq_len'].numpy(), table.type_tag.tolist(),
                                table.o_tag, table.cls_tag, table.sep_tag)
    return dict(logits=logits, loss=loss, pred_ids=pred, margin=margin, pairs=pr)


def _estimator(tmp_path, B, L, seed, **extra):
    (tmp_path / "bert_config.json").write_text(json.dumps(SMALL_BERT))
    feats = synthetic.msra_batch(B, L, vocab=SMALL_BERT['vocab_size'], seed=seed)
    est = engine.Estimator("bert_mrc", dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), mrc_query_ids=_query_ids(),
                                            **extra))
    est.evaluate(feats)                                     # creates the variables
    est.store.vars["logits/kernel"].mul_(8.0)               # O(1) logits: non-trivial decisions
    est.store.touch()
    return est, feats


def _cuda_logits(est, dev):
    """The plugin's logits [B*T, L, 3], by the same calls as build_graph."""
    from chinesener_b200.model import _blocks, bert_mrc
    from chinesener_b200.tools import layer
    table = mrc.device_table(est.params)
    B, L = dev['token_ids'].shape
    with variables.use_store(est.store):
        pr = ops.mrc_pairs(dev['token_ids'], dev['seq_len'], table.query_ids, table.query_len, table.type_tag, table.L2,
                           table.sep_id)
        pr['mask'].total_tokens = table.pair_tokens(dev['mask'])
        hidden = _blocks.bert_sequence({'token_ids': pr['ids'], 'mask': pr['mask'], 'segment_ids': pr['segment_ids']},
                                       est.params, False)
        rows = bert_mrc.sentence_rows(hidden, pr['align'], B * table.T, L, False)
        return layer.dense(rows, 3, 'logits')


def test_bert_mrc_predict_and_eval_match_oracle(tmp_path):
    B, L = 6, 48
    est, feats = _estimator(tmp_path, B, L, seed=5)
    table = mrc.device_table(est.params)
    assert table.names == ['ORG', 'PER', 'LOC'] and table.query_lens == [22, 10, 20]
    assert est.store.vars["logits/kernel"].shape == (768, 3) and "crf_layer/transitions" not in est.store.vars
    out = est.evaluate(feats)
    pred = est.predict(feats)['pred_ids'].numpy()
    np.testing.assert_array_equal(out['pred_ids'].numpy(), pred)
    dev = est.to_device(feats)
    lg = _cuda_logits(est, dev)
    # pred_ids = the merge of the CUDA logits, bit for bit
    seq_len = feats['seq_len'].numpy()
    own, own_margin = oracle_merge(lg.cpu().numpy(), seq_len, table.type_tag.tolist(), table.o_tag, table.cls_tag,
                                   table.sep_tag)
    near = own_margin <= 1e-4
    assert (pred[~near] == own[~near]).all()
    w = est.store.state_dict()
    ref = bert_mrc_oracle(w, feats, table, emulate_bf16=True)
    pair_len = torch.from_numpy(ref['pairs']['seq_len'])
    valid = torch.arange(L)[None, :] < pair_len[:, None]
    scale = ref['logits'][valid].abs().max().item()
    err = (lg.cpu().double() - ref['logits'])[valid].abs().max().item()
    print(f"bert_mrc: max|logit - oracle(bf16-emulated)| over the valid positions = {err:.2e} (scale {scale:.2f})")
    assert err < 4e-3 * scale
    loss_ref = float(ref['loss'])
    assert abs(out['loss'] - loss_ref) < 5e-3 * abs(loss_ref), (out['loss'], loss_ref)
    sure = ref['margin'] > 1e-2
    assert sure.mean() > 0.5
    np.testing.assert_array_equal(pred[sure], ref['pred_ids'][sure])
    claimed = (pred >= 2) & (pred <= 7)
    assert claimed.any()                                    # the merge does pick entity tags
    # a second call is bit-identical
    assert torch.equal(est.predict(feats)['pred_ids'], torch.from_numpy(pred))
    assert est.evaluate(feats)['loss'] == out['loss']


def test_bert_mrc_predict_has_no_device_sync(tmp_path):
    """PREDICT sizes the packed pairs from the host counts of Estimator.to_device: no device-to-host synchronisation."""
    B, L = 16, 64
    est, feats = _estimator(tmp_path, B, L, seed=9)
    dev = est.to_device(feats)
    assert dev['mask'].nonempty_rows == int((feats['seq_len'] > 0).sum())
    ref = est.predict_device(dev)                           # warm: weight packs, workspaces
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        pred = est.predict_device(dev)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(pred, ref)
    # stacked batches carry the counts too
    parts = [synthetic.msra_batch(5, L, vocab=SMALL_BERT['vocab_size'], seed=s) for s in (1, 2)]
    parts[1]['seq_len'][0] = 0
    parts[1]['mask'][0] = 0
    parts[1]['token_ids'][0] = 0
    stacked = est.stack_to_device(parts)
    assert stacked['mask'].nonempty_rows == 9 and stacked['mask'].total_tokens == sum(int(p['mask'].sum()) for p in parts)
    torch.cuda.set_sync_debug_mode('error')
    try:
        pred = est.predict_device(stacked)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    expect = torch.cat([est.predict(p)['pred_ids'] for p in parts])
    assert (pred.cpu() == expect).float().mean().item() > 0.99      # row counts differ: GEMM tilings may differ
    assert (pred.cpu()[5] == 0).all()


# --------------------------------------------------------------------------- TRAIN
CFG_TRAIN = {'vocab_size': 1500, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
             'intermediate_size': 3072, 'max_position_embeddings': 128, 'type_vocab_size': 2, 'initializer_range': 0.02}


def _train_est(tmp_path, dropout=0.0, bert_dropout=0.0, B=4, L=32):
    cfg = dict(CFG_TRAIN, hidden_dropout_prob=bert_dropout, attention_probs_dropout_prob=bert_dropout)
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    feats = synthetic.msra_batch(B, L, vocab=CFG_TRAIN['vocab_size'], seed=21)
    feats['seq_len'][1] = 0                                 # an empty sentence: empty pairs
    feats['mask'][1] = 0
    feats['token_ids'][1] = 0
    feats['label_ids'][1] = 0
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), embedding_dropout=dropout,
                  mrc_query_ids=_query_ids(vocab=CFG_TRAIN['vocab_size']))
    return engine.Estimator("bert_mrc", params), feats


@pytest.mark.parametrize("packed", [True, False])
def test_bert_mrc_gradients_match_oracle_autograd(tmp_path, packed, monkeypatch):
    from chinesener_b200.tools import layer as _layer
    monkeypatch.setattr(_layer, "TRAIN_PACK", packed)
    est, feats = _train_est(tmp_path)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(4.0)
    est.store.touch()
    table = mrc.device_table(est.params)
    w = est.store.state_dict()
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    ref = bert_mrc_oracle(wd, feats, table)
    ref['loss'].backward()
    ref_loss = float(ref['loss'].detach())
    dev = est.to_device(feats)
    with variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, pred = est.build_graph(dev, None, est.params, True)
        tape.backward()
    assert abs(float(loss) - ref_loss) < 2e-2 * max(1.0, abs(ref_loss))
    assert pred.shape == feats['label_ids'].shape and pred.dtype == torch.int32
    worst = {}
    grads = {k: v.grad for k, v in wd.items()}
    gscale = max(g.abs().max().item() for n, g in grads.items() if g is not None and "pooler" not in n)
    for name, g_ref in grads.items():
        if g_ref is None or "pooler" in name:
            continue
        g = est.store.grads[name].cpu().double()
        scale = max(g_ref.abs().max().item(), 1e-3 * gscale)
        worst[name] = (g - g_ref).abs().max().item() / scale
    bad = {k: v for k, v in worst.items() if v > 8e-2}
    print("max relative gradient error:", max(worst.values()), "over", len(worst), "variables")
    assert not bad, bad


def test_bert_mrc_training_reduces_loss(tmp_path):
    est, feats = _train_est(tmp_path, dropout=0.1, bert_dropout=0.1)
    est.params.update(lr=5e-5, num_train_steps=100, warmup_ratio=0.1)
    losses = [float(est.train_step(feats)) for _ in range(12)]
    print("bert_mrc losses:", ["%.3f" % v for v in losses])
    assert np.isfinite(losses).all(), losses
    assert losses[-1] < 0.8 * losses[0], losses


# --------------------------------------------------------------------------- driver and InferHelper
def test_driver_writes_bert_mrc_prediction_pickle(tmp_path):
    from chinesener_b200 import main as driver
    from test_main_driver_gpu import L as DRIVER_L, _setup
    root, pre = _setup(tmp_path)
    vocab = ['[PAD]', '[UNK]', '[CLS]', '[SEP]'] + sorted(set(''.join(mrc.DEFAULT_QUERIES.values())))
    with open(os.path.join(pre, 'vocab.txt'), 'w', encoding='utf-8') as f:      # the default queries are tokenized with it
        f.write('\n'.join(vocab) + '\n')
    cfg_path = os.path.join(pre, 'bert_config.json')
    cfg = json.load(open(cfg_path))
    cfg['vocab_size'] = max(cfg['vocab_size'], len(vocab))
    json.dump(cfg, open(cfg_path, 'w'))
    with pytest.warns(UserWarning):                    # no BERT checkpoint in pretrain_dir: random init
        s = driver.main(['--model_name', 'bert_mrc', '--data', 'msra', '--data_dir', os.path.join(root, 'msra'),
                         '--checkpoint_root', str(tmp_path / 'ckpt'), '--pretrain_dir', pre, '--epoch_size', '2',
                         '--batch_size', '4'])
    assert s['n_predict'] == 24 and s['history']['final_step'] == 16 * 2 // 4
    path = os.path.join(root, 'msra', 'bert_mrc_predict.pkl')
    pred = pickle.load(open(path, 'rb'))
    assert len(pred) == 24
    assert all(p['pred_ids'].shape == (DRIVER_L,) and p['pred_ids'].dtype == np.int32 for p in pred)
    assert all(int(p['pred_ids'].max()) < 10 and int(p['pred_ids'].min()) >= 0 for p in pred)
    assert np.isfinite(s['entity_micro_f1'])
    from chinesener_b200.data.records import NerDataset
    idx2tag = NerDataset(os.path.join(root, 'msra'), 4, 2, 'bert_mrc').params['idx2tag']
    tag_rep, ent_rep = evaluation.SingleEval(path, idx2tag).gen_report()
    assert 0.0 <= ent_rep['micro avg']['f1-score'] <= 1.0 and 'weighted avg' in tag_rep


def test_infer_helper_batch_equals_single_sentences(tmp_path):
    from chinesener_b200.data.tokenizer import FullTokenizer
    from chinesener_b200.inference import InferHelper, TAG2IDX
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "warmup_features.json"), encoding="utf8"))
    vocab = dict(gold["bert_vocab_subset"])
    vocab.setdefault("[UNK]", 100)
    (tmp_path / "bert_config.json").write_text(json.dumps(dict(SMALL_BERT, vocab_size=21128)))
    params = dict(synthetic.data_params(150), pretrain_dir=str(tmp_path), mrc_query_ids=_query_ids(vocab=21128))
    est = engine.Estimator("bert_mrc", params)
    helper = InferHelper(150, TAG2IDX, "bert_mrc", FullTokenizer(vocab), estimator=est)
    text = gold["text"]
    helper.infer(text)                                           # first call creates the variables
    est.store.vars["logits/kernel"].mul_(8.0)
    est.store.touch()
    texts = [text, text[:7], text[3:30], text[::2]]
    single = [dict(helper.infer(t)) for t in texts]
    batch = [dict(e) for e in helper.infer_batch(texts)]
    assert batch == single
