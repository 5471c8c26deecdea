"""GPU: the bert_ce plugin (reference model/bert_ce.py) and its softmax-head kernel ner_token_xent.

  * kernel vs float64: first-max argmax bit-exact at every position, masked token-mean loss within 1e-5 relative,
    d_logits within 1e-6 of float64 autograd and exactly 0 past seq_len, deterministic;
  * plugin PREDICT / EVAL vs a float64 restatement of bert_ce (padded BertModel, label projection, masked CE, argmax at
    every position): logits at ALL positions within 4e-3 of the logit scale of the bf16-emulated restatement, and the
    pinned property of the reference's prediction pickles — [PAD] positions carry real, mostly non-zero tags;
  * TRAIN: every variable's gradient against float64 autograd (packed and padded encoder), and a short AdamW run;
  * the command-line driver writes bert_ce_predict.pkl.
"""
import ctypes
import json
import os
import pickle

import numpy as np
import pytest
import torch

from chinesener_b200 import _lib, autodiff, engine, evaluation, ops, synthetic, variables
from oracle import nn as onn

pytestmark = pytest.mark.gpu

SMALL_BERT = {'vocab_size': 3000, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
              'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02}


# --------------------------------------------------------------------------- float64 restatement of model/bert_ce.py
def masked_token_xent(logits, labels, seq_len):
    """tools/loss.py cross_entropy_loss: mean over t < seq_len of logsumexp(z) - z[y]; 0 without tokens."""
    B, L, _ = logits.shape
    valid = torch.arange(L)[None, :] < seq_len.long()[:, None]
    ce = torch.logsumexp(logits, -1) - logits.gather(-1, labels.long().clamp(min=0)[..., None])[..., 0]
    n = int(valid.sum())
    return (ce * valid).sum() / n if n > 0 else (ce * 0.0).sum()


def bert_ce_oracle(w, features, params, dtype=torch.float64, emulate_bf16=False, gelu_variant="tanh"):
    """model/bert_ce.py (eval mode): padded BertModel -> dense 'logits' (bf16-rounded sequence output when emulating the
    bf16 path, as for bert_crf) -> masked token-mean CE, pred_ids = first argmax at every position."""
    seq = onn.bert_encoder(w, features["token_ids"], features["mask"], features["segment_ids"],
                           num_layers=params.get("num_hidden_layers", 12), num_heads=params.get("num_attention_heads", 12),
                           dtype=dtype, gelu_variant=gelu_variant, emulate_bf16=emulate_bf16)
    logits = onn.dense(onn._rb(seq, emulate_bf16), w["logits/kernel"].to(dtype), w["logits/bias"].to(dtype))
    loss = masked_token_xent(logits, features["label_ids"], features["seq_len"])
    pred = logits.detach().argmax(-1).to(torch.int32).numpy()
    return dict(logits=logits, loss=float(loss.detach()), pred_ids=pred)


# --------------------------------------------------------------------------- kernel
def _kernel_case(B, L, K, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn((B, L, K), generator=g) * 3.0
    if K > 1:                                   # tied maxima: the lowest index must win
        flat = z.view(-1, K)
        rows = torch.arange(0, flat.shape[0], 3)
        flat[rows, K - 1] = flat[rows].max(-1).values + 1.0
        flat[rows, K // 2] = flat[rows, K - 1]
        flat[rows[::2], 0] = flat[rows[::2], K - 1]
    labels = torch.randint(0, K, (B, L), generator=g, dtype=torch.int32)
    lens = torch.randint(0, L + 1, (B,), generator=g, dtype=torch.int32)
    if B >= 3:
        lens[0], lens[1], lens[2] = 0, 1, L
    else:
        lens[0] = L
    return z, labels, lens


def _reference(z, labels, lens, d_loss=1.0):
    zd = z.double().requires_grad_(True)
    loss = masked_token_xent(zd, labels, lens)
    (loss * d_loss).backward()
    return float(loss.detach()), zd.grad


@pytest.mark.parametrize("B,L,K", [(1, 1, 1), (7, 33, 10), (64, 128, 10), (5, 150, 32), (3, 16, 7)])
def test_token_xent_matches_float64(B, L, K):
    z, labels, lens = _kernel_case(B, L, K, seed=B * 1000 + L * 10 + K)
    zc, lc, nc = z.cuda(), labels.cuda(), lens.cuda()
    pred, loss, dz = ops.token_xent(zc, lc, nc, want_grad=True)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(pred.cpu().numpy(), np.argmax(z.numpy(), axis=-1).astype(np.int32))
    ref_loss, ref_grad = _reference(z, labels, lens)
    assert abs(float(loss) - ref_loss) <= 1e-5 * max(abs(ref_loss), 1e-30), (float(loss), ref_loss)
    dz = dz.cpu()
    assert (dz.double() - ref_grad).abs().max().item() < 1e-6
    past = torch.arange(L)[None, :] >= lens.long()[:, None]
    assert (dz[past] == 0).all()
    # argmax only (PREDICT) and loss only (EVAL) launches agree with the fused one
    pred_only, no_loss, no_grad = ops.token_xent(zc)
    assert no_loss is None and no_grad is None
    assert torch.equal(pred_only, pred)
    _, loss_only, _ = ops.token_xent(zc, lc, nc, want_pred=False)
    assert float(loss_only) == float(loss)
    # d_loss scales the gradient
    _, _, dz_half = ops.token_xent(zc, lc, nc, want_grad=True, d_loss=0.5)
    _, ref_half = _reference(z, labels, lens, d_loss=0.5)
    assert (dz_half.cpu().double() - ref_half).abs().max().item() < 1e-6


def test_token_xent_is_deterministic():
    z, labels, lens = _kernel_case(4096, 128, 10, seed=3)
    zc, lc, nc = z.cuda(), labels.cuda(), lens.cuda()
    _, l1, g1 = ops.token_xent(zc, lc, nc, want_grad=True)
    _, l2, g2 = ops.token_xent(zc, lc, nc, want_grad=True)
    assert l1.cpu().numpy().tobytes() == l2.cpu().numpy().tobytes()
    assert torch.equal(g1, g2)
    ref_loss, _ = _reference(z, labels, lens)
    assert abs(float(l1) - ref_loss) <= 1e-5 * abs(ref_loss)


def test_token_xent_empty_batch_and_limits():
    z, labels, _ = _kernel_case(5, 12, 10, seed=9)
    zc, lc = z.cuda(), labels.cuda()
    pred, loss, dz = ops.token_xent(zc, lc, torch.zeros(5, dtype=torch.int32, device='cuda'), want_grad=True)
    assert float(loss) == 0.0 and not dz.any()
    assert torch.equal(pred.cpu(), torch.from_numpy(np.argmax(z.numpy(), -1).astype(np.int32)))
    with pytest.raises(_lib.NerB200Error, match="unsupported"):
        ops.token_xent(torch.zeros((2, 4, 33), device='cuda'))
    h = _lib.lib()
    assert h.ner_token_xent(ctypes.c_void_p(zc.data_ptr()), None, None, ctypes.c_void_p(pred.data_ptr()), None, None, 1.0,
                            None, 5, 12, 33, None) == -2


# --------------------------------------------------------------------------- plugin PREDICT / EVAL
def _estimator(tmp_path, B, L, seed, **extra):
    (tmp_path / "bert_config.json").write_text(json.dumps(SMALL_BERT))
    feats = synthetic.msra_batch(B, L, vocab=SMALL_BERT['vocab_size'], seed=seed)
    est = engine.Estimator("bert_ce", dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), **extra))
    est.evaluate(feats)                                     # creates the variables
    est.store.vars["logits/kernel"].mul_(8.0)               # O(1) logits: non-trivial argmax
    est.store.touch()
    return est, feats


def _cuda_logits(est, dev):
    from chinesener_b200.model import _blocks
    from chinesener_b200.tools import layer
    prec0 = layer.BERT_PRECISION
    layer.BERT_PRECISION = est.params.get('bert_precision', prec0)
    try:
        with variables.use_store(est.store):
            seq = _blocks.bert_sequence(dev, est.params, False, packed=False)
            return layer.dense(seq, est.params['label_size'], 'logits')
    finally:
        layer.BERT_PRECISION = prec0


def test_bert_ce_predict_and_eval_match_oracle(tmp_path):
    B, L = 6, 48
    est, feats = _estimator(tmp_path, B, L, seed=5)
    out = est.evaluate(feats)
    pred = est.predict(feats)['pred_ids'].numpy()
    np.testing.assert_array_equal(out['pred_ids'].numpy(), pred)
    lg = _cuda_logits(est, est.to_device(feats)).cpu()
    # pred_ids = argmax of the CUDA logits at every position, bit for bit
    np.testing.assert_array_equal(pred, np.argmax(lg.numpy(), -1).astype(np.int32))
    w = est.store.state_dict()
    p = dict(est.params, num_hidden_layers=2, num_attention_heads=12)
    ref = bert_ce_oracle(w, feats, p, emulate_bf16=True)
    scale = max(1.0, ref['logits'].abs().max().item())
    err = (lg.double() - ref['logits']).abs().max().item()
    print(f"bert_ce: max|logit - oracle(bf16-emulated)| over all positions = {err:.2e} (scale {scale:.2f})")
    assert err < 4e-3 * scale
    agree = (pred == ref['pred_ids']).mean()
    assert agree > 0.99, agree
    pad = (torch.arange(L)[None, :] >= feats['seq_len'][:, None]).numpy()
    assert pad.any() and (pred[pad] != 0).any()             # [PAD] positions carry real tags, as the reference's pickles
    assert abs(out['loss'] - ref['loss']) < 5e-3 * abs(ref['loss']), (out['loss'], ref['loss'])


def test_bert_ce_fp32_precision_mode(tmp_path):
    """params['bert_precision'] = 'fp32' runs through the fp32-accurate encoder unchanged: logits at the real tokens within
    1e-3 of the float64 restatement, and the loss with them.  That encoder's attention writes zero rows for [PAD] queries,
    so its [PAD] tags are not the reference's (the bf16 path above computes them)."""
    B, L = 6, 48
    est, feats = _estimator(tmp_path, B, L, seed=5, bert_precision='fp32')
    out = est.evaluate(feats)
    lg = _cuda_logits(est, est.to_device(feats)).cpu()
    np.testing.assert_array_equal(out['pred_ids'].numpy(), np.argmax(lg.numpy(), -1).astype(np.int32))
    w = est.store.state_dict()
    ref = bert_ce_oracle(w, feats, dict(est.params, num_hidden_layers=2, num_attention_heads=12), emulate_bf16=False)
    valid = torch.arange(L)[None, :] < feats['seq_len'][:, None]
    err = (lg.double() - ref['logits'])[valid].abs().max().item()
    print(f"bert_ce fp32 mode: max|logit - fp64 oracle| over the real tokens = {err:.2e}")
    assert err < 1e-3
    assert abs(out['loss'] - ref['loss']) < 1e-3 * max(1.0, abs(ref['loss']))


# --------------------------------------------------------------------------- TRAIN
CFG_TRAIN = {'vocab_size': 1500, 'hidden_size': 768, 'num_hidden_layers': 2, 'num_attention_heads': 12,
             'intermediate_size': 3072, 'max_position_embeddings': 128, 'type_vocab_size': 2, 'initializer_range': 0.02}


def _train_est(tmp_path, dropout=0.0, bert_dropout=0.0, B=4, L=32):
    cfg = dict(CFG_TRAIN, hidden_dropout_prob=bert_dropout, attention_probs_dropout_prob=bert_dropout)
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    feats = synthetic.msra_batch(B, L, vocab=CFG_TRAIN['vocab_size'], seed=21)
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), embedding_dropout=dropout)
    return engine.Estimator("bert_ce", params), feats


@pytest.mark.parametrize("packed", [True, False])
def test_bert_ce_gradients_match_oracle_autograd(tmp_path, packed, monkeypatch):
    from chinesener_b200.tools import layer as _layer
    monkeypatch.setattr(_layer, "TRAIN_PACK", packed)
    est, feats = _train_est(tmp_path)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(4.0)
    est.store.touch()
    w = est.store.state_dict()
    assert "crf_layer/transitions" not in w and {"logits/kernel", "logits/bias"} <= set(w)
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    seq = onn.bert_encoder(wd, feats['token_ids'], feats['mask'], feats['segment_ids'], num_layers=2, num_heads=12,
                           dtype=torch.float64)
    ref_loss_t = masked_token_xent(seq @ wd['logits/kernel'] + wd['logits/bias'], feats['label_ids'], feats['seq_len'])
    ref_loss_t.backward()
    ref_loss = float(ref_loss_t.detach())
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


def test_bert_ce_training_reduces_loss(tmp_path):
    est, feats = _train_est(tmp_path, dropout=0.1, bert_dropout=0.1)
    # the 'logit' group trains at 500x lr (TRAIN_PARAMS): 2e-4 makes the loss of this 4-sentence batch oscillate
    est.params.update(lr=5e-5, num_train_steps=100, warmup_ratio=0.1)
    losses = [float(est.train_step(feats)) for _ in range(12)]
    print("bert_ce losses:", ["%.3f" % v for v in losses])
    assert np.isfinite(losses).all(), losses
    assert losses[-1] < 0.8 * losses[0], losses


# --------------------------------------------------------------------------- driver
def test_driver_writes_bert_ce_prediction_pickle(tmp_path):
    from chinesener_b200 import main as driver
    from test_main_driver_gpu import L as DRIVER_L, _setup
    root, pre = _setup(tmp_path)
    with pytest.warns(UserWarning):                    # no BERT checkpoint in pretrain_dir: random init
        s = driver.main(['--model_name', 'bert_ce', '--data', 'msra', '--data_dir', os.path.join(root, 'msra'),
                         '--checkpoint_root', str(tmp_path / 'ckpt'), '--pretrain_dir', pre, '--epoch_size', '2',
                         '--batch_size', '4'])
    assert s['n_predict'] == 24 and s['history']['final_step'] == 16 * 2 // 4
    path = os.path.join(root, 'msra', 'bert_ce_predict.pkl')
    pred = pickle.load(open(path, 'rb'))
    assert len(pred) == 24
    assert all(p['pred_ids'].shape == (DRIVER_L,) and p['pred_ids'].dtype == np.int32 for p in pred)
    assert all(int(p['pred_ids'].max()) < 10 and int(p['pred_ids'].min()) >= 0 for p in pred)
    assert np.isfinite(s['entity_micro_f1'])
    from chinesener_b200.data.records import NerDataset
    idx2tag = NerDataset(os.path.join(root, 'msra'), 4, 2, 'bert_ce').params['idx2tag']
    assert max(idx2tag) < 10
    tag_rep, ent_rep = evaluation.SingleEval(path, idx2tag).gen_report()
    assert 0.0 <= ent_rep['micro avg']['f1-score'] <= 1.0 and 'weighted avg' in tag_rep
