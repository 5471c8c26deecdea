"""GPU: the bert_dice plugin (reference model/bert_dice.py) and its softmax-head kernel ner_token_dice.

  * kernel vs float64: first-max argmax bit-exact at every position, masked token-mean Dice loss within 1e-5 relative,
    d_logits within 1e-5 of max|ref| of float64 autograd, exactly 0 past seq_len and finite on rows saturated by +40;
    K = 1 against its closed values; deterministic;
  * plugin: the same pred_ids as bert_ce on one state dict, EVAL loss vs the bf16-emulated float64 restatement for two
    values of dice_gamma, every variable's gradient vs float64 autograd (packed and padded encoder), a short AdamW run;
  * the command-line driver writes bert_dice_predict.pkl.
"""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from chinesener_b200 import autodiff, engine, evaluation, ops, synthetic, variables
from oracle import nn as onn

from test_bert_ce_gpu import CFG_TRAIN, _estimator, _kernel_case, bert_ce_oracle

pytestmark = pytest.mark.gpu


# --------------------------------------------------------------------------- float64 restatement of tools/loss.py dice_loss
def masked_token_dice(logits, labels, seq_len, alpha, gamma):
    """Mean over t < seq_len of sum_k l_k, l_y = (1 - q_y) / (q_y + 1 + gamma), l_k = q_k / (q_k + gamma), q = (1-p)^alpha p;
    0 without tokens.  1 - p_k is exp(logsumexp_{i != k} z - logsumexp z): finite and accurate (and differentiable) on
    confident rows, where 1 - p rounds to 0."""
    B, L, K = logits.shape
    valid = torch.arange(L)[None, :] < seq_len.long()[:, None]
    lse = torch.logsumexp(logits, -1, keepdim=True)
    p = torch.exp(logits - lse)
    others = logits[..., None, :].expand(B, L, K, K).masked_fill(torch.eye(K, dtype=torch.bool), float('-inf'))
    u = torch.exp(torch.logsumexp(others, -1) - lse)
    q = u ** alpha * p
    onehot = torch.nn.functional.one_hot(labels.long().clamp(min=0), K).bool()
    tok = torch.where(onehot, (1 - q) / (q + 1 + gamma), q / (q + gamma)).sum(-1)
    n = int(valid.sum())
    return (tok * valid).sum() / n if n > 0 else (tok * 0.0).sum()


def _dice_case(B, L, K, seed):
    """bert_ce's kernel inputs (tied maxima, seq_len 0 / 1 / L) plus rows saturated by +40, on the label and off it."""
    z, labels, lens = _kernel_case(B, L, K, seed)
    flat, lab = z.view(-1, K), labels.view(-1)
    rows = torch.arange(1, flat.shape[0], 5)
    flat[rows, lab[rows].long()] += 40.0                                  # confident and right
    rows = torch.arange(2, flat.shape[0], 7)
    flat[rows, ((lab[rows] + 1) % K).long()] += 40.0                      # confident and wrong (right when K = 1)
    return z, labels, lens


def _reference(z, labels, lens, alpha, gamma, d_loss=1.0):
    zd = z.double().requires_grad_(True)
    loss = masked_token_dice(zd, labels, lens, alpha, gamma)
    (loss * d_loss).backward()
    return float(loss.detach()), zd.grad


KERNEL_CASES = [(B, L, K, alpha, 1.0) for (B, L, K) in [(7, 33, 10), (64, 128, 10), (5, 150, 32), (3, 16, 7)]
                for alpha in (0.0, 0.5, 1.0, 2.0)] + [(64, 128, 10, 1.0, 0.1)]


@pytest.mark.parametrize("B,L,K,alpha,gamma", KERNEL_CASES)
def test_token_dice_matches_float64(B, L, K, alpha, gamma):
    z, labels, lens = _dice_case(B, L, K, seed=B * 1000 + L * 10 + K)
    zc, lc, nc = z.cuda(), labels.cuda(), lens.cuda()
    pred, loss, dz = ops.token_dice(zc, lc, nc, alpha, gamma, want_grad=True)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(pred.cpu().numpy(), np.argmax(z.numpy(), axis=-1).astype(np.int32))
    ref_loss, ref_grad = _reference(z, labels, lens, alpha, gamma)
    assert torch.isfinite(ref_grad).all()
    assert abs(float(loss) - ref_loss) <= 1e-5 * abs(ref_loss), (float(loss), ref_loss)
    dz = dz.cpu()
    assert torch.isfinite(dz).all()
    gscale = ref_grad.abs().max().item()
    err = (dz.double() - ref_grad).abs().max().item()
    assert err <= 1e-5 * gscale, (err, gscale)
    past = torch.arange(L)[None, :] >= lens.long()[:, None]
    assert (dz[past] == 0).all()
    # the loss-only (EVAL) launch gives the fused launch's loss bit for bit
    _, loss_only, no_grad = ops.token_dice(zc, lc, nc, alpha, gamma, want_pred=False)
    assert no_grad is None and float(loss_only) == float(loss)
    # d_loss scales the gradient
    _, _, dz_half = ops.token_dice(zc, lc, nc, alpha, gamma, want_grad=True, d_loss=0.5)
    _, ref_half = _reference(z, labels, lens, alpha, gamma, d_loss=0.5)
    assert (dz_half.cpu().double() - ref_half).abs().max().item() <= 1e-5 * gscale * 0.5


@pytest.mark.parametrize("alpha", [0.0, 0.5, 1.0, 2.0])
def test_token_dice_single_class(alpha):
    """K = 1: p = 1, u = 0, so a token's loss is 1 / (1 + gamma) for alpha > 0 and 0 for alpha = 0, and the gradient 0."""
    gamma = 0.5
    z = torch.randn(3, 5, 1, device='cuda') * 3.0
    labels = torch.zeros(3, 5, dtype=torch.int32, device='cuda')
    lens = torch.tensor([0, 1, 5], dtype=torch.int32, device='cuda')
    pred, loss, dz = ops.token_dice(z, labels, lens, alpha, gamma, want_grad=True)
    assert not pred.any()
    assert float(loss) == pytest.approx(1.0 / (1.0 + gamma) if alpha > 0 else 0.0, rel=1e-6, abs=0.0)
    assert not dz.any()


def test_token_dice_is_deterministic():
    z, labels, lens = _dice_case(4096, 128, 10, seed=3)
    zc, lc, nc = z.cuda(), labels.cuda(), lens.cuda()
    _, l1, g1 = ops.token_dice(zc, lc, nc, 1.0, 1.0, want_grad=True)
    _, l2, g2 = ops.token_dice(zc, lc, nc, 1.0, 1.0, want_grad=True)
    assert l1.cpu().numpy().tobytes() == l2.cpu().numpy().tobytes()
    assert torch.equal(g1, g2)
    ref_loss, _ = _reference(z, labels, lens, 1.0, 1.0)
    assert abs(float(l1) - ref_loss) <= 1e-5 * abs(ref_loss)
    # an all-empty batch: loss 0, gradient 0, argmax still at every position
    pred, loss, dz = ops.token_dice(zc[:5], lc[:5], torch.zeros(5, dtype=torch.int32, device='cuda'), want_grad=True)
    assert float(loss) == 0.0 and not dz.any()
    assert torch.equal(pred.cpu(), torch.from_numpy(np.argmax(z[:5].numpy(), -1).astype(np.int32)))


# --------------------------------------------------------------------------- plugin PREDICT / EVAL
def test_bert_dice_predict_and_eval_match_oracle(tmp_path):
    B, L = 6, 48
    ce, feats = _estimator(tmp_path, B, L, seed=5)                       # bert_ce, O(1) logits
    est = engine.Estimator("bert_dice", dict(ce.params), store=ce.store)
    assert est.params['dice_alpha'] == 1.0 and est.params['dice_gamma'] == 1.0
    pred = est.predict(feats)['pred_ids'].numpy()
    np.testing.assert_array_equal(pred, ce.predict(feats)['pred_ids'].numpy())
    out = est.evaluate(feats)
    np.testing.assert_array_equal(out['pred_ids'].numpy(), pred)
    pad = (torch.arange(L)[None, :] >= feats['seq_len'][:, None]).numpy()
    assert pad.any() and (pred[pad] != 0).any()             # [PAD] positions carry real tags, as bert_ce's
    w = est.store.state_dict()
    ref = bert_ce_oracle(w, feats, dict(est.params, num_hidden_layers=2, num_attention_heads=12), emulate_bf16=True)
    losses = {}
    for gamma in (1.0, 0.1):
        est.params['dice_gamma'] = gamma
        ref_loss = float(masked_token_dice(ref['logits'], feats['label_ids'], feats['seq_len'], 1.0, gamma))
        losses[gamma] = est.evaluate(feats)['loss']
        print(f"bert_dice gamma={gamma}: EVAL loss {losses[gamma]:.6f}, restatement {ref_loss:.6f}")
        assert abs(losses[gamma] - ref_loss) < 5e-3 * abs(ref_loss), (gamma, losses[gamma], ref_loss)
    assert abs(losses[1.0] - losses[0.1]) > 0.1 * losses[1.0]


# --------------------------------------------------------------------------- TRAIN
def _train_est(tmp_path, dropout=0.0, bert_dropout=0.0, B=4, L=32):
    cfg = dict(CFG_TRAIN, hidden_dropout_prob=bert_dropout, attention_probs_dropout_prob=bert_dropout)
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    feats = synthetic.msra_batch(B, L, vocab=CFG_TRAIN['vocab_size'], seed=21)
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), embedding_dropout=dropout)
    return engine.Estimator("bert_dice", params), feats


@pytest.mark.parametrize("packed", [True, False])
def test_bert_dice_gradients_match_oracle_autograd(tmp_path, packed, monkeypatch):
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
    ref_loss_t = masked_token_dice(seq @ wd['logits/kernel'] + wd['logits/bias'], feats['label_ids'], feats['seq_len'],
                                   est.params['dice_alpha'], est.params['dice_gamma'])
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


def test_bert_dice_training_reduces_loss(tmp_path):
    est, feats = _train_est(tmp_path, dropout=0.1, bert_dropout=0.1)
    est.params.update(lr=5e-5, num_train_steps=100, warmup_ratio=0.1)
    # measured on an H100: 1.02 -> 0.50 by step 5, then flat — with alpha = 1 a token whose softmax is one-hot costs
    # 1 / (2 + gamma) = 0.5 and has no gradient left; the 0.8 bar leaves room for the dropout noise of step 1
    losses = [float(est.train_step(feats)) for _ in range(12)]
    print("bert_dice losses:", ["%.4f" % v for v in losses])
    assert np.isfinite(losses).all(), losses
    assert losses[-1] < 0.8 * losses[0], losses


# --------------------------------------------------------------------------- driver
def test_driver_writes_bert_dice_prediction_pickle(tmp_path):
    from chinesener_b200 import main as driver
    from test_main_driver_gpu import L as DRIVER_L, _setup
    root, pre = _setup(tmp_path)
    with pytest.warns(UserWarning):                    # no BERT checkpoint in pretrain_dir: random init
        s = driver.main(['--model_name', 'bert_dice', '--data', 'msra', '--data_dir', os.path.join(root, 'msra'),
                         '--checkpoint_root', str(tmp_path / 'ckpt'), '--pretrain_dir', pre, '--epoch_size', '2',
                         '--batch_size', '4'])
    assert s['n_predict'] == 24 and s['history']['final_step'] == 16 * 2 // 4
    path = os.path.join(root, 'msra', 'bert_dice_predict.pkl')
    pred = pickle.load(open(path, 'rb'))
    assert len(pred) == 24
    assert all(p['pred_ids'].shape == (DRIVER_L,) and p['pred_ids'].dtype == np.int32 for p in pred)
    assert all(int(p['pred_ids'].max()) < 10 and int(p['pred_ids'].min()) >= 0 for p in pred)
    assert all(set(p) >= {'pred_ids', 'label_ids', 'tokens'} for p in pred)
    assert np.isfinite(s['entity_micro_f1'])
    from chinesener_b200.data.records import NerDataset
    idx2tag = NerDataset(os.path.join(root, 'msra'), 4, 2, 'bert_dice').params['idx2tag']
    tag_rep, ent_rep = evaluation.SingleEval(path, idx2tag).gen_report()
    assert 0.0 <= ent_rep['micro avg']['f1-score'] <= 1.0 and 'weighted avg' in tag_rep
